"""Torch-facing API: put / get CUDA tensors through the object store with the fused kernels.

    store = TensorStore(cluster.client)
    store.batch_put(["act/0", "act/1"], [t0, t1])                  # BBH64 digest fused into the copy
    store.put("kv/layer3", kv_fp16, pack_fp8=True)                  # block-scaled MXFP8 on the wire / in the slab
    t = store.get("kv/layer3")                                      # verified + unpacked fp16 tensor

    store.put_bundle("ckpt/step100", model.state_dict())            # many tensors, one object and one `#meta`
    store.get_bundle_into("ckpt/step100", model.state_dict())       # loaded in place into the parameters

Tensor metadata (dtype, shape, packing) travels in a small side object `<key>#meta`.
"""
from __future__ import annotations

import json
from typing import Optional, Sequence

import numpy as np
import torch

from .. import _bb

_DTYPES = {str(d).replace("torch.", ""): d for d in (torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float16,
                                                     torch.bfloat16, torch.float32, torch.float64, torch.bool)}
# dtypes MXFP8 packing takes, and the wide type the kernels read / write them as
_MX_WIDE = {torch.bfloat16: _bb.MxWide.BF16, torch.float16: _bb.MxWide.F16, torch.float32: _bb.MxWide.F32}
# Smallest page that put_blocks / get_blocks_into move with the paged device calls; smaller pages take index_select +
# put and get + index_copy_.  bench/paged_bench.py, 256 blocks of a bf16 cache on one H100 80GB HBM3 at 700 W: the paged
# calls' kernel time equals a plain transfer's at every page size, but each call carries ~0.5-0.8 ms of host work, so
# they win from 32 KiB pages (XXH3 put 1.65 vs 2.10 ms, get 1.35 vs 2.32 ms at 512 MiB, and no temporary) and lose at
# 16 KiB and below (8 KiB: 1.1 vs 0.8 ms).
PAGED_MIN_PAGE_BYTES = 32 << 10
# The same for packed (MXFP8) objects, whose alternative route (index_select + packed put, get + index_copy_) runs the
# pack or unpack kernel as well.  bench/fp8_paged_bench.py, 256 blocks of a bf16 cache on one H100 80GB HBM3 at 700 W,
# median ms: the paged calls win at 32 KiB pages (put 1.19 vs 1.81, get 1.30 vs 1.76, and no 512 MiB temporary) and at
# 16 KiB (put 0.96 vs 1.02, get 0.99 vs 1.10), and lose from 8 KiB down (put 0.98 vs 0.80, get 0.92 vs 0.84).
FP8_PAGED_MIN_PAGE_BYTES = 16 << 10
# The same for partial restores of packed objects (get_blocks_into with `blocks`), whose alternative route also runs a
# whole-object index_select.  bench/paged_partial_bench.py, 256 stored blocks of a cache [32, 2, 2048, h, 8, 128] on one
# H100 80GB HBM3 at 700 W, median ms of the paged unpack vs get + index_select + index_copy_: at 32 KiB pages it wins from
# k = 128 restored blocks on (bf16 1.16 vs 1.70, fp32 1.24 vs 1.32; k = 256: 1.41 vs 2.61) and is within 0.15 ms at
# k = 16 (bf16 0.89 vs 0.94, fp32 1.02 vs 0.88); at 16 KiB it loses at k = 16 in every dtype (bf16 1.04 vs 0.81, fp32
# 1.07 vs 0.78) and for fp32 also at k = 128 (1.27 vs 1.14), so the crossover is 32 KiB, not FP8_PAGED_MIN_PAGE_BYTES.
# Unpacked partial restores keep PAGED_MIN_PAGE_BYTES: the same run shows them winning at 32 KiB (XXH3 k = 128: 1.30 vs
# 1.80 ms) and losing at 16 KiB for k = 16 and at 8 KiB and below for every k.
FP8_PARTIAL_MIN_PAGE_BYTES = 32 << 10
# Smallest page that put_layer_blocks / get_layer_blocks_into move with block ids that stay on the device
# (batch_put_device_blocks / batch_get_device_blocks); smaller pages take index_select + stack + put and get +
# index_copy_.  bench/layer_blocks_bench.py, 32 per-layer bf16 caches [2, 2048, h, 8, 128] with 256 blocks selected, on
# one H100 80GB HBM3 at 700 W, two runs: the device route beats index_select + stack + put / get + index_copy_ at every
# page size measured, 32, 16, 8 and 4 KiB, with XXH3 and without a checksum (4 KiB put 0.80-0.86 vs 1.49-2.24 ms
# median, get 0.86-1.00 vs 1.47-1.70).  Smaller pages were not measured, so they keep the other route.  DESIGN.md
# section 5 has the numbers.
LAYER_BLOCKS_MIN_PAGE_BYTES = 4 << 10
# The same for packed (MXFP8) objects (batch_put_device_fp8_blocks / batch_get_device_fp8_blocks), whose other route runs
# the pack or unpack kernel as well.  The same benchmark, packed bf16 (every page size) and fp16 / fp32 (32 KiB): the
# device route wins everywhere measured too (bf16 4 KiB put 0.78-0.95 vs 1.83-2.03 ms, get 0.95-0.97 vs 1.59-1.74).
FP8_LAYER_BLOCKS_MIN_PAGE_BYTES = 4 << 10
# Shortest in-page row that the paged and block-id calls move when a block's page is rows inside it (a head slice of a
# KV cache, _block_pages); shorter rows take index_select + put and get + index_copy_.  bench/sliced_blocks_bench.py,
# 256 blocks of bf16 NHD / HND caches (2-32 MiB objects) on one H100 80GB HBM3 at 700 W, 15 calls: the transfer kernel
# with rows of 256 bytes and more takes 0.9-1.2x the time of a contiguous paged transfer of the same bytes (1 head,
# 256 B rows: put 0.029 vs 0.024 ms, get 0.027 vs 0.027), with 128 B rows 1.2-1.4x (put 0.030 vs 0.022, get 0.029 vs
# 0.025), and at 128 B the call loses to index_select + put by more than at 256 B (median put 0.62 vs 0.44 ms, get 0.73
# vs 0.53).  At these object sizes every route is host-bound (~0.5 ms a call) and the min-max spreads overlap, but the
# row route's median is 0.05-0.25 ms above index_select + put / get + index_copy_ at every row size measured, 256 B and
# more included: below this threshold it loses by more, above it it still does not win on time, only in memory (no
# temporary as large as the selection).  Where that host time goes was not measured, nor were objects large enough for
# the paged route to win on time (the 512 MiB workloads of PAGED_MIN_PAGE_BYTES).
PAGED_MIN_ROW_BYTES = 256


def _stored_dtype(m) -> torch.dtype:
    """The dtype a stored tensor is returned as: its own, packed or not (packed metas always record it)."""
    return _DTYPES[m["dtype"]]


def _by_dtype(idx, dtype_of) -> dict:
    """idx grouped by dtype_of(i), in order: one native call per wide type."""
    groups = {}
    for i in idx:
        groups.setdefault(dtype_of(i), []).append(i)
    return groups


def _check(what: str, keys, ecs, fallback: bool = False) -> None:
    """RuntimeError naming the first items whose code is not OK; with `fallback`, NOT_IMPLEMENTED is no error either
    (the packed calls refuse with it what a fallback route then takes)."""
    bad = [(k, e) for k, e in zip(keys, ecs) if e != _bb.ErrorCode.OK and not (fallback and e == _bb.ErrorCode.NOT_IMPLEMENTED)]
    if bad:
        raise RuntimeError(f"{what} failed: {bad[:3]}")


def _meta(dtype: torch.dtype, shape, packed: bool) -> bytes:
    """The `#meta` record of a tensor; a packed one also records its element count padded to whole 32-element MX blocks."""
    n = torch.Size(shape).numel()
    meta = {"dtype": str(dtype).replace("torch.", ""), "shape": list(shape), "packed": "mxfp8" if packed else None, "numel": n}
    if packed:
        meta["padded_numel"] = (n + 31) // 32 * 32
    return json.dumps(meta).encode()


def _elem_rows(es: int, rows, n: int):
    """(width, pitch, rows) in elements of `es` bytes: byte rows (see TensorStore._source_rows), or n contiguous elements
    as one row when rows is None."""
    return (rows[0] // es, rows[1] // es, rows[2]) if rows is not None else (n, n, 1)


class TensorStore:
    def __init__(self, client, config: Optional["_bb.WorkerConfig"] = None):
        self.client = client
        self.config = config or _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1,
                                                 preferred_classes=[_bb.StorageClass.RAM_GPU])

    @staticmethod
    def _stream() -> int:
        return torch.cuda.current_stream().cuda_stream

    def _meta_cfg(self):
        return _bb.WorkerConfig(replication_factor=self.config.replication_factor, max_workers_per_copy=1, ttl_ms=self.config.ttl_ms,
                                enable_soft_pin=self.config.enable_soft_pin, checksum=_bb.ChecksumAlgo.CRC32C)

    def _put_metas(self, keys: list, metas: list) -> None:
        ecs = self.client.batch_put([k + "#meta" for k in keys], metas, self._meta_cfg())
        if any(e != _bb.ErrorCode.OK for e in ecs):
            raise RuntimeError("meta put failed")

    def _packed(self, what: str, keys: list, idx: list, dtype_of, call) -> list:
        """One native call per dtype for the packed items idx: call(group, element size, wide) returns the group's error
        codes.  RuntimeError for a code other than OK or NOT_IMPLEMENTED; returns the items refused with NOT_IMPLEMENTED,
        in call order, for the caller's fallback."""
        refused = []
        for dt, grp in _by_dtype(idx, dtype_of).items():
            ecs = call(grp, dt.itemsize, _MX_WIDE[dt])
            _check(what, [keys[i] for i in grp], ecs, fallback=True)
            refused += [i for i, e in zip(grp, ecs) if e == _bb.ErrorCode.NOT_IMPLEMENTED]
        return refused

    def _whole(self, keys: list, idx: list, device, fn) -> None:
        """fn(i, t) for each item of idx with its whole stored tensor t from batch_get: the route of the items no device
        call above took."""
        if idx:
            for i, t in zip(idx, self.batch_get([keys[i] for i in idx], device)):
                fn(i, t)

    def _fp8_whole(self, m) -> bool:
        """A packed object the fused unpack reads: unpadded, a whole number of 32-element MX blocks."""
        return m["packed"] == "mxfp8" and m["padded_numel"] == m["numel"] and self.client.device_fp8_eligible(m["numel"])

    # ------------------------------------------------------------------ put
    @staticmethod
    def _fusable_fp8_cfg(cfg) -> bool:
        """Up to 3 copies (one tile pass of the fused pack fans out to every replica), each copy in one shard."""
        return 1 <= cfg.replication_factor <= 3 and cfg.max_workers_per_copy == 1

    def _fused_fp8_ok(self, t: torch.Tensor, cfg) -> bool:
        """Pack fused into the put kernel: bf16, fp16 or fp32, a whole number of 32-element MX blocks, a fusable config."""
        return t.dtype in _MX_WIDE and self.client.device_fp8_eligible(t.numel()) and self._fusable_fp8_cfg(cfg) and t.data_ptr() % 16 == 0

    @staticmethod
    def _source_rows(t: torch.Tensor):
        """(width, pitch, rows) in bytes when `t`'s elements are rows of `width` bytes every `pitch` bytes from
        t.data_ptr() in row-major order, else None: a contiguous block of trailing dims gives the width and the leading dims
        must collapse to one stride, the pitch.  This covers `narrow` along any dim of a contiguous tensor and `t[::k]`;
        transposed, overlapping or otherwise permuted layouts give None."""
        dims = [(n, s) for n, s in zip(t.shape, t.stride()) if n != 1]
        width = t.element_size()
        while dims and dims[-1][1] * t.element_size() == width:  # the trailing contiguous block
            width *= dims.pop()[0]
        if not dims:
            return width, width, 1
        pitch, rows = dims[-1][1] * t.element_size(), 1
        for k, (n, s) in enumerate(dims):
            if k + 1 < len(dims) and s != dims[k + 1][1] * dims[k + 1][0]:
                return None
            rows *= n
        return (width, pitch, rows) if pitch >= width else None

    def _gatherable(self, t: torch.Tensor):
        """The (width, pitch, rows) of a non-contiguous CUDA tensor that the fused put can read in place: rows (see
        _source_rows), a 16-byte aligned start and a row gap that is a multiple of 16 bytes.  None for any other tensor;
        those are made contiguous on the device first, which beats staging them through the host."""
        if not t.is_cuda or t.is_contiguous() or t.numel() == 0 or t.data_ptr() % 16:
            return None
        r = self._source_rows(t)
        return r if r is not None and (r[2] == 1 or (r[1] - r[0]) % 16 == 0) else None

    def batch_put(self, keys: Sequence[str], tensors: Sequence[torch.Tensor], pack_fp8: bool = False, config=None) -> None:
        """Stores each tensor under its key.  A slice of a larger CUDA tensor whose elements are rows -- `W[:, a:b]`, `kv[:,
        :, h0:h1, :]`, `t[::k]` -- is read in place by the fused put kernel (batch_put_device_strided) when its start is
        16-byte aligned and its row gap a multiple of 16 bytes; no contiguous copy is made.  With pack_fp8 such a slice
        whose element count is a whole number of 32-element MX blocks is gathered the same way by the fused pack kernel
        (batch_put_device_fp8_strided) when the config is fusable.  Other layouts are made contiguous first.  The stored
        object is that of `t.contiguous()` either way.

        pack_fp8 takes bf16, fp16 and fp32 tensors (TypeError for any other dtype, before anything is stored): each is
        packed from its own values, with no bf16 copy, and gets return it in its own dtype.  A batch that mixes dtypes
        makes one native call per dtype."""
        cfg = config or self.config
        keys = list(keys)
        tensors = list(tensors)
        if pack_fp8:
            bad = [(k, t.dtype) for k, t in zip(keys, tensors) if t.dtype not in _MX_WIDE]
            if bad:
                raise TypeError(f"MXFP8 packing takes bfloat16, float16 and float32 tensors, not {bad[:3]}")
        rows = [self._gatherable(t) for t in tensors]
        if pack_fp8:  # only slices the fused pack kernel can take are gathered
            rows = [r if r is not None and self._fused_fp8_ok(t, cfg) else None for t, r in zip(tensors, rows)]
        tensors = [t if r is not None else t.contiguous() for t, r in zip(tensors, rows)]
        # objects the fused kernel can take go through batch_put_device_fp8 (bf16 read once, packed bytes on the wire,
        # digest of the packed object from the tensor cores); the rest are packed first (unfused path below)
        fused = [i for i, t in enumerate(tensors) if t.is_cuda and self._fused_fp8_ok(t, cfg)] if pack_fp8 else []
        if fused:
            def call(grp, es, wide):
                fk, ptrs = [keys[i] for i in grp], [tensors[i].data_ptr() for i in grp]
                if any(rows[i] is not None for i in grp):
                    # one call and one launch: contiguous tensors go as one row each
                    shapes = [_elem_rows(es, rows[i], tensors[i].numel()) for i in grp]
                    return self.client.batch_put_device_fp8_strided(fk, ptrs, *map(list, zip(*shapes)), cfg, self._stream(), wide=wide)
                return self.client.batch_put_device_fp8(fk, ptrs, [tensors[i].numel() for i in grp], cfg, self._stream(), wide=wide)

            refused = set(self._packed("fused fp8 put", keys, fused, lambda i: tensors[i].dtype, call))
            done = [i for grp in _by_dtype(fused, lambda i: tensors[i].dtype).values() for i in grp if i not in refused]
            if done:
                self._put_metas([keys[i] for i in done], [_meta(tensors[i].dtype, tensors[i].shape, True) for i in done])
            done = set(done)
            rest = [i for i in range(len(keys)) if i not in done]
            # a gathered slice the fused put refused (its placement is not one GPU-fabric shard per copy) is made
            # contiguous and packed first, like any other
            keys, tensors = [keys[i] for i in rest], [tensors[i].contiguous() for i in rest]
            rows = [None] * len(keys)
            if not keys:
                return
        payloads, metas, keep = [], [], []
        for t in tensors:
            assert t.is_cuda, "TensorStore moves CUDA tensors (host data: use client.put)"
            metas.append(_meta(t.dtype, t.shape, pack_fp8))
            if pack_fp8:
                n = t.numel()
                npad = (n + 31) // 32 * 32
                src = t.view(-1)
                if npad != n:
                    src = torch.cat([src, torch.zeros(npad - n, dtype=t.dtype, device=t.device)])
                packed = torch.empty(_bb.mxfp8_packed_bytes(npad), dtype=torch.uint8, device=t.device)
                _bb.mxfp8_pack(src.data_ptr(), npad, packed.data_ptr(), self._stream(), wide=_MX_WIDE[t.dtype])
                keep.append(src)
                t = packed
            assert t.data_ptr() % 16 == 0, "tensor storage must be 16-byte aligned"
            payloads.append(t)
        ptrs, sizes = [p.data_ptr() for p in payloads], [p.numel() * p.element_size() for p in payloads]
        if any(r is not None for r in rows):
            # one call and one launch for the whole batch: the other tensors go as one row each (pack_fp8 has no rows)
            shapes = [_elem_rows(1, r, n) for r, n in zip(rows, sizes)]
            ecs = self.client.batch_put_device_strided(list(keys), ptrs, *map(list, zip(*shapes)), cfg, self._stream())
        else:
            ecs = self.client.batch_put_device(list(keys), ptrs, sizes, cfg, self._stream())
        _check("put", keys, ecs)
        self._put_metas(keys, metas)

    def put(self, key: str, tensor: torch.Tensor, pack_fp8: bool = False, config=None) -> None:
        self.batch_put([key], [tensor], pack_fp8, config)

    # ------------------------------------------------------------------ blocks of a paged cache
    @staticmethod
    def _block_dim(key: str, cache: torch.Tensor, dim: int) -> int:
        """`dim` as a dimension of `cache`, negative dims counting from the end; IndexError out of range, as index_select."""
        if not -cache.dim() <= dim < cache.dim():
            raise IndexError(f"{key}: dim {dim} out of range for {cache.dim()} dimensions")
        return dim % cache.dim()

    @staticmethod
    def _block_ids(key: str, ids, size: int, what: str = "block ids") -> np.ndarray:
        """`ids` (a list or an integer tensor) as a 1-D int64 numpy array; a CUDA tensor is copied to the host once, which
        synchronises with its stream.  IndexError for an id outside [0, size); `what` names the argument in errors."""
        if isinstance(ids, torch.Tensor):
            if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
                raise TypeError(f"{key}: {what} must be a 1-D integer list or tensor")
            a = ids.to(device="cpu", dtype=torch.int64).numpy()
        else:
            a = np.asarray(list(ids))
            if a.size == 0:
                a = a.astype(np.int64)
            if a.dtype.kind not in "iu":
                raise TypeError(f"{key}: {what} must be a 1-D integer list or tensor")
            a = a.astype(np.int64)
        if a.ndim != 1:
            raise TypeError(f"{key}: {what} must be a 1-D integer list or tensor")
        if a.size and (a.min() < 0 or a.max() >= size):
            raise IndexError(f"{key}: {what} must lie in [0, {size})")
        return a

    @staticmethod
    def _block_pages(cache: torch.Tensor, dim: int, ids: np.ndarray, min_page: Optional[int] = None):
        """(page addresses, page bytes, rows) of cache.index_select(dim, ids) for the paged device calls, or None when they
        should not move it.  Page (o, k) is cache[o..., ids[k]] over the dims after `dim`, in index_select order (outer
        index major): those dims must be one contiguous block (rows None), or rows inside the block, rows =
        (row_width, row_pitch) in bytes as _source_rows gives them for one block (a head slice of a KV cache: a trailing
        contiguous block gives the width, the other dims collapse to one pitch), with rows of at least PAGED_MIN_ROW_BYTES
        and a gap between them of a multiple of 16 bytes.  The page (its dense bytes) must be a multiple of 16 bytes and at
        least `min_page` bytes (by default PAGED_MIN_PAGE_BYTES; FP8_PAGED_MIN_PAGE_BYTES for packed objects), the outer dims
        must collapse to one positive stride, the blocks must not overlap one another over their true extent (no zero or
        negative strides: an expanded cache takes the fallback) and every page must be 16-byte aligned.  The addresses are
        a numpy int64 array, built without a loop per page."""
        if not cache.is_cuda or cache.numel() == 0 or ids.size == 0:
            return None
        es, shape, stride = cache.element_size(), cache.shape, cache.stride()
        inner = [(n, s) for n, s in zip(shape[dim + 1:], stride[dim + 1:]) if n != 1]
        width = es
        while inner and inner[-1][1] * es == width:  # the trailing contiguous block
            width *= inner.pop()[0]
        page, extent, rows = width, width, None
        if inner:  # rows inside the block: the other dims must collapse to one pitch
            if any(s != s2 * n2 for (_, s), (n2, s2) in zip(inner, inner[1:])):
                return None
            n, pitch = int(np.prod([n for n, _ in inner], dtype=np.int64)), inner[-1][1] * es
            if pitch <= width or (pitch - width) % 16 or width < PAGED_MIN_ROW_BYTES:
                return None
            page, extent, rows = n * width, (n - 1) * pitch + width, (width, pitch)
        if page % 16 or page < (PAGED_MIN_PAGE_BYTES if min_page is None else min_page):
            return None
        outer = [(n, s) for n, s in zip(shape[:dim], stride[:dim]) if n != 1]
        if any(s != s2 * n2 for (_, s), (n2, s2) in zip(outer, outer[1:])):
            return None
        n_outer = int(np.prod([n for n, _ in outer], dtype=np.int64))
        o_step = outer[-1][1] * es if outer else 0
        b_step = stride[dim] * es
        # disjoint blocks: every (outer, block) step positive and at least the extent of the smaller steps' blocks
        for n, step in sorted([(n, st) for n, st in ((n_outer, o_step), (shape[dim], b_step)) if n > 1], key=lambda t: t[1]):
            if step < extent:
                return None
            extent = step * (n - 1) + extent
        addrs = (cache.data_ptr() + np.arange(n_outer, dtype=np.int64)[:, None] * o_step + ids[None, :] * b_step).reshape(-1)
        if (addrs & 15).any():
            return None
        return addrs, page, rows

    @staticmethod
    def _rows_in(rows, es: int):
        """A _block_pages row pattern in elements of `es` bytes (the packed calls count in elements), None kept."""
        return None if rows is None else (rows[0] // es, rows[1] // es)

    def batch_put_blocks(self, keys: Sequence[str], caches: Sequence[torch.Tensor], ids: Sequence, dim: int = 0, pack_fp8: bool = False,
                         config=None) -> None:
        """Stores `caches[i].index_select(dim, ids[i])` under keys[i], with the usual `#meta`, so get, get_into, get_rows
        and get_slice read it unchanged: the blocks of a request in a paged KV cache, all layers at once, as one object.
        IndexError for an id out of range, before anything is stored.

        When the cache is a CUDA tensor whose dims after `dim` form one contiguous block of a multiple of 16 bytes and at
        least PAGED_MIN_PAGE_BYTES (32 KiB, where the paged calls start to beat index_select), whose outer dims collapse
        to one stride, whose blocks do not overlap and whose pages are 16-byte aligned, the blocks are read in place by
        the paged put (batch_put_device_paged): no index_select temporary, no extra device pass.  Any other layout takes
        index_select and batch_put.

        With pack_fp8 (bf16, fp16 and fp32 caches; TypeError for any other dtype, before anything is stored), a cache of
        that layout with pages of at least FP8_PAGED_MIN_PAGE_BYTES, whose selected element count is a whole number of
        32-element MX blocks, under a fusable config (up to 3 copies, one shard each), is packed in place by the paged
        pack kernel (batch_put_device_fp8_paged): no wide temporary.  The stored object is that of
        put(index_select(...), pack_fp8=True).  Items the fused kernel refuses (NOT_IMPLEMENTED: an unfusable placement)
        and other layouts take index_select and batch_put.  IndexError for a dim out of range.  A CUDA `ids` tensor is
        copied to the host once, which synchronises."""
        keys, caches, ids = list(keys), list(caches), list(ids)
        if not len(keys) == len(caches) == len(ids):
            raise ValueError("keys, caches and ids differ in length")
        cfg = config or self.config
        if pack_fp8:
            bad = [(k, c.dtype) for k, c in zip(keys, caches) if c.dtype not in _MX_WIDE]
            if bad:
                raise TypeError(f"MXFP8 packing takes bfloat16, float16 and float32 tensors, not {bad[:3]}")
        dims = [self._block_dim(k, c, dim) for k, c in zip(keys, caches)]
        idx = [self._block_ids(k, b, c.shape[d]) for k, c, b, d in zip(keys, caches, ids, dims)]
        shapes = []
        for c, d, b in zip(caches, dims, idx):
            shapes.append(list(c.shape))
            shapes[-1][d] = b.size
        min_page = FP8_PAGED_MIN_PAGE_BYTES if pack_fp8 else PAGED_MIN_PAGE_BYTES
        pages = [self._block_pages(c, d, b, min_page) for c, d, b in zip(caches, dims, idx)]
        if pack_fp8:  # the fused pack takes whole MX blocks under a fusable config
            pages = [p if p is not None and self._fusable_fp8_cfg(cfg) and self.client.device_fp8_eligible(torch.Size(s).numel()) else None
                     for p, s in zip(pages, shapes)]
        paged = [i for i, p in enumerate(pages) if p is not None]
        if paged and pack_fp8:
            def call(grp, es, wide):
                return self.client.batch_put_device_fp8_paged([keys[i] for i in grp], [pages[i][0] for i in grp],
                                                              [pages[i][1] // es for i in grp], cfg, self._stream(), wide=wide,
                                                              rows=[self._rows_in(pages[i][2], es) for i in grp])

            refused = set(self._packed("paged fp8 put", keys, paged, lambda i: caches[i].dtype, call))
            paged = [i for grp in _by_dtype(paged, lambda i: caches[i].dtype).values() for i in grp if i not in refused]
        elif paged:
            ecs = self.client.batch_put_device_paged([keys[i] for i in paged], [pages[i][0] for i in paged], [pages[i][1] for i in paged],
                                                     cfg, self._stream(), rows=[pages[i][2] for i in paged])
            _check("paged put", [keys[i] for i in paged], ecs)
        if paged:
            self._put_metas([keys[i] for i in paged], [_meta(caches[i].dtype, shapes[i], pack_fp8) for i in paged])
        done = set(paged)
        rest = [i for i in range(len(keys)) if i not in done]
        if rest:
            self.batch_put([keys[i] for i in rest], [caches[i].index_select(dims[i], torch.from_numpy(idx[i]).to(caches[i].device)) for i in rest],
                           pack_fp8, config)

    def put_blocks(self, key: str, cache: torch.Tensor, ids, dim: int = 0, pack_fp8: bool = False, config=None) -> None:
        """Stores `cache.index_select(dim, ids)` under `key` (see batch_put_blocks)."""
        self.batch_put_blocks([key], [cache], [ids], dim, pack_fp8, config)

    @staticmethod
    def _sparse_table(addrs: np.ndarray, blocks: np.ndarray, n_stored: int) -> np.ndarray:
        """The page table over the whole stored object of a partial restore: `addrs` are the pages of the cache blocks the
        selected stored blocks land in (_block_pages, outer index major, blocks.size per outer index), placed at those
        blocks' positions among the n_stored blocks per outer index; every other entry is 0, a page the get does not
        store."""
        table = np.zeros((addrs.size // blocks.size, n_stored), dtype=np.int64)
        table[:, blocks] = addrs.reshape(-1, blocks.size)
        return table.reshape(-1)

    def batch_get_blocks_into(self, keys: Sequence[str], caches: Sequence[torch.Tensor], ids: Sequence, dim: int = 0,
                              blocks: Optional[Sequence] = None) -> list:
        """`caches[i].index_copy_(dim, ids[i], stored)` for the tensor stored under keys[i]: restores a request's KV blocks
        into whatever free blocks the allocator handed out.  No element of a cache outside the selected blocks is written.
        Returns `caches`.

        With `blocks`, only some stored blocks are restored: `caches[i].index_copy_(dim, ids[i], stored.index_select(dim,
        blocks[i]))`, blocks[i] indexing the stored tensor's `dim` -- a new request reusing the first k blocks of a stored
        prefix (blocks=range(k)), or the evicted blocks of a request refilled while the rest stay resident.  blocks=None is
        every stored block in order.

        Every check comes before any transfer, so a cache is untouched after an error: KeyError for a missing key,
        TypeError unless the cache dtype is the stored dtype or for ids or blocks that are not integers, ValueError unless
        the stored shape is the index_select shape (with blocks: unless it equals the cache shape outside `dim` and
        len(blocks[i]) == len(ids[i])), for a cache that is not a CUDA tensor on the current device and for duplicate ids
        or blocks, IndexError for an id, a block or a dim out of range.  An empty selection with blocks moves nothing.

        Caches of the layout batch_put_blocks reads in place take the paged get (batch_get_device_paged), which stores
        each tile straight into its pages (RuntimeError unless the stored object fills the table); packed whole-block
        tensors with pages of at least FP8_PAGED_MIN_PAGE_BYTES (FP8_PARTIAL_MIN_PAGE_BYTES with blocks) take the paged
        unpack (batch_get_device_fp8_paged), which unpacks each tile straight into its pages.  With blocks, the table covers the whole stored object and the pages of
        the stored blocks not selected are 0 (not stored): the whole object is still read and verified, but there is no
        temporary and no index_select.  Other layouts, padded packed tensors, and packed objects the fused kernel refuses
        (NOT_IMPLEMENTED: an unfusable placement) take a get followed by index_select and index_copy_.  CUDA `ids` or
        `blocks` tensors are copied to the host once, which synchronises."""
        keys, caches, ids = list(keys), list(caches), list(ids)
        if not len(keys) == len(caches) == len(ids):
            raise ValueError("keys, caches and ids differ in length")
        if blocks is not None:
            blocks = list(blocks)
            if len(blocks) != len(keys):
                raise ValueError("keys and blocks differ in length")
        metas = self._metas(keys)
        dev = torch.cuda.current_device()
        dims = [self._block_dim(k, c, dim) for k, c in zip(keys, caches)]
        idx, sel = [], []  # sel[i]: the selected stored blocks, None for all of them
        for j, (k, m, c, b, d) in enumerate(zip(keys, metas, caches, ids, dims)):
            if c.dtype != _stored_dtype(m):
                raise TypeError(f"{k}: cache is {c.dtype}, the stored tensor {_stored_dtype(m)}")
            t = self._block_ids(k, b, c.shape[d])
            s = None
            if blocks is None:
                shape = list(c.shape)
                shape[d] = t.size
                if shape != m["shape"]:
                    raise ValueError(f"{k}: the stored tensor has shape {m['shape']}, the selected blocks {shape}")
            else:
                stored = m["shape"]
                if len(stored) != c.dim() or any(a != n for e, (a, n) in enumerate(zip(stored, c.shape)) if e != d):
                    raise ValueError(f"{k}: the stored tensor has shape {stored}, the cache {list(c.shape)}: they differ outside dim {d}")
                s = self._block_ids(k, blocks[j], stored[d], "blocks")
                if s.size != t.size:
                    raise ValueError(f"{k}: {s.size} blocks for {t.size} ids")
            if not c.is_cuda or c.device.index != dev:
                raise ValueError(f"{k}: cache must be a CUDA tensor on cuda:{dev}, not {c.device}")
            if np.unique(t).size != t.size:
                raise ValueError(f"{k}: duplicate block ids")
            if s is not None and np.unique(s).size != s.size:
                raise ValueError(f"{k}: duplicate blocks")
            idx.append(t)
            sel.append(s)
        live = [i for i in range(len(keys)) if sel[i] is None or sel[i].size]  # an empty selection moves nothing
        # packed whole-block objects take the paged unpack; padded ones cannot fill whole pages
        fp8 = [self._fp8_whole(m) for m in metas]
        pages = [None] * len(keys)
        for i in live:
            if fp8[i] or not metas[i]["packed"]:
                fp8_min = FP8_PAGED_MIN_PAGE_BYTES if sel[i] is None else FP8_PARTIAL_MIN_PAGE_BYTES
                pages[i] = self._block_pages(caches[i], dims[i], idx[i], fp8_min if fp8[i] else PAGED_MIN_PAGE_BYTES)
            if pages[i] is not None and sel[i] is not None:
                pages[i] = (self._sparse_table(pages[i][0], sel[i], metas[i]["shape"][dims[i]]), pages[i][1], pages[i][2])

        def call(grp, es, wide):
            return self.client.batch_get_device_fp8_paged([keys[i] for i in grp], [pages[i][0] for i in grp], [pages[i][1] // es for i in grp],
                                                          self._stream(), wide=wide, rows=[self._rows_in(pages[i][2], es) for i in grp])

        for i in self._packed("paged fp8 get", keys, [i for i, p in enumerate(pages) if p is not None and fp8[i]], lambda i: caches[i].dtype, call):
            pages[i] = None  # get + index_copy_ below
        paged = [i for i, p in enumerate(pages) if p is not None and not fp8[i]]
        if paged:
            ecs, sizes = self.client.batch_get_device_paged([keys[i] for i in paged], [pages[i][0] for i in paged],
                                                            [pages[i][1] for i in paged], self._stream(), rows=[pages[i][2] for i in paged])
            # the stored object must fill the table: a shorter one would leave the last blocks as they were; those are
            # named after the items that failed
            short = [f"{n} bytes stored, {pages[i][0].size * pages[i][1]} selected" if e == _bb.ErrorCode.OK and n != pages[i][0].size * pages[i][1]
                     else _bb.ErrorCode.OK for i, e, n in zip(paged, ecs, sizes)]
            _check("paged get", [keys[i] for i in paged] * 2, list(ecs) + short)

        def restore(i, t):
            if sel[i] is not None:
                t = t.index_select(dims[i], torch.from_numpy(sel[i]).to(t.device))
            caches[i].index_copy_(dims[i], torch.from_numpy(idx[i]).to(caches[i].device), t)

        self._whole(keys, [i for i in live if pages[i] is None], None, restore)
        return caches

    def get_blocks_into(self, key: str, cache: torch.Tensor, ids, dim: int = 0, blocks=None) -> torch.Tensor:
        """`cache.index_copy_(dim, ids, stored)`, or with `blocks` `cache.index_copy_(dim, ids, stored.index_select(dim,
        blocks))`, for the tensor stored under `key` (see batch_get_blocks_into)."""
        return self.batch_get_blocks_into([key], [cache], [ids], dim, None if blocks is None else [blocks])[0]

    # ------------------------------------------------------------------ blocks of per-layer caches, ids on the device
    @staticmethod
    def _layers(key: str, caches) -> tuple:
        """(list of caches, stacked): one tensor, or a list of same-shape, same-dtype tensors on one device (one per layer,
        stacked along a new dim 0).  ValueError otherwise."""
        if isinstance(caches, torch.Tensor):
            return [caches], False
        caches = list(caches)
        if not caches or any(c.shape != caches[0].shape or c.dtype != caches[0].dtype or c.device != caches[0].device for c in caches):
            raise ValueError(f"{key}: caches must be one tensor or a non-empty list of same-shape, same-dtype tensors on one device")
        return caches, True

    @staticmethod
    def _device_ids(t, device) -> bool:
        """Whether `t` is a 1-D CUDA int32 or int64 tensor on `device`: ids the device route reads where they are."""
        return isinstance(t, torch.Tensor) and t.is_cuda and t.device == device and t.dim() == 1 and t.dtype in (torch.int32, torch.int64)

    def _device_blocks(self, layers: list, dim: int, ids: torch.Tensor, sel: Optional[torch.Tensor], n_stored: int, packed: bool = False):
        """The DeviceBlocks of `layers` (index_select(dim, ids) of each, layer-major), with the id tensors it points to, or
        None when the device route should not move them: the layout batch_put_blocks reads in place, pages of at least
        LAYER_BLOCKS_MIN_PAGE_BYTES (FP8_LAYER_BLOCKS_MIN_PAGE_BYTES when `packed`, whose pages are then counted in
        elements), a block stride of a multiple of 16 bytes, and layers that do not overlap one another (a get into
        aliased layers would store two blocks into one page at once; the fallback's per-layer index_copy_ is ordered).
        The slice addresses are computed from the shapes and strides alone; the ids are never read here."""
        if ids.numel() == 0:
            return None
        # the layers share shape and dtype; those that share strides too differ only in their base address
        es = layers[0].element_size()
        first = self._block_pages(layers[0], dim, np.zeros(1, dtype=np.int64), FP8_LAYER_BLOCKS_MIN_PAGE_BYTES if packed else LAYER_BLOCKS_MIN_PAGE_BYTES)
        stride = layers[0].stride(dim) * es
        if first is None or stride % 16 or any(c.stride() != layers[0].stride() or c.data_ptr() % 16 for c in layers):
            return None
        extent = (1 + sum((n - 1) * st for n, st in zip(layers[0].shape, layers[0].stride()))) * es
        starts = sorted(c.data_ptr() for c in layers)
        if any(a + extent > b for a, b in zip(starts, starts[1:])):
            return None
        base = layers[0].data_ptr()
        wide = ids.dtype == torch.int64 or (sel is not None and sel.dtype == torch.int64)
        dt = torch.int64 if wide else torch.int32
        ids = ids.to(dt).contiguous()
        sel = None if sel is None else sel.to(dt).contiguous()
        outer = np.concatenate([first[0] + (c.data_ptr() - base) for c in layers])
        unit = es if packed else 1
        rows = self._rows_in(first[2], unit) or (0, 0)
        b = _bb.DeviceBlocks(outer, ids.data_ptr(), ids.numel(), layers[0].shape[dim], stride, first[1] // unit, id_bytes=dt.itemsize,
                             sel=0 if sel is None else sel.data_ptr(), n_stored=n_stored if sel is not None else 0,
                             row_width=rows[0], row_pitch=rows[1])
        return b, (ids, sel)

    @staticmethod
    def _verdicts(keys: list, items: list, ecs: list) -> None:
        """Raises for the items the device refused on their ids: IndexError for an id or block out of range, ValueError for
        a repeated one (a get's); RuntimeError for any other code but OK."""
        for i, e in zip(items, ecs):
            if e == _bb.ErrorCode.VALUE_OUT_OF_RANGE:
                raise IndexError(f"{keys[i]}: block ids or blocks out of range")
            if e == _bb.ErrorCode.INVALID_ARGUMENT:
                raise ValueError(f"{keys[i]}: duplicate block ids or blocks")
        _check("layer blocks transfer", [keys[i] for i in items], ecs)

    def batch_put_layer_blocks(self, keys: Sequence[str], caches: Sequence, ids: Sequence, dim: int = 0, pack_fp8: bool = False,
                               config=None) -> None:
        """Stores `torch.stack([c.index_select(dim, ids[i]) for c in caches[i]])` under keys[i] -- one object for a
        request's blocks in every layer of an engine that keeps one KV tensor per layer -- with the usual `#meta`, so get,
        get_rows, get_slice, and get_blocks_into on a stacked cache read it unchanged.  caches[i] may also be a single
        tensor, stored as `index_select(dim, ids[i])` alone.  ValueError for caches of different shapes, dtypes or
        devices, IndexError for a dim out of range, TypeError for pack_fp8 with a dtype other than bf16, fp16 or fp32,
        all before anything is stored.

        CUDA int32 or int64 `ids` on the caches' device stay there: when every cache has the layout batch_put_blocks
        reads in place with pages of at least LAYER_BLOCKS_MIN_PAGE_BYTES, the transfer engine builds the page table on
        the device from the ids (batch_put_device_blocks) and the put kernel reads the blocks in place, with no host
        synchronisation.  With pack_fp8, caches of that layout with pages of at least FP8_LAYER_BLOCKS_MIN_PAGE_BYTES,
        whose selected element count is a whole number of MX blocks, under a fusable config (as put_blocks), are packed as
        the pages are read (batch_put_device_fp8_blocks, one call per dtype).  Then an id out of range is found on the
        device, after the transfer: IndexError is raised after the call, that key stores nothing (no object, no `#meta`),
        and the other keys of the batch complete.  This differs from put_blocks, which checks ids before any transfer.
        Layers that overlap one another take the fallback.

        Every other case -- host ids, other layouts, smaller pages, and placements the device route cannot take
        (NOT_IMPLEMENTED) -- checks the ids on the host first (IndexError before that key is stored; a CUDA ids tensor is
        copied to the host, which synchronises) and takes index_select + stack + batch_put."""
        keys, caches, ids = list(keys), list(caches), list(ids)
        if not len(keys) == len(caches) == len(ids):
            raise ValueError("keys, caches and ids differ in length")
        cfg = config or self.config
        layers = [self._layers(k, c) for k, c in zip(keys, caches)]
        if pack_fp8:
            bad = [(k, ls[0].dtype) for k, (ls, _) in zip(keys, layers) if ls[0].dtype not in _MX_WIDE]
            if bad:
                raise TypeError(f"MXFP8 packing takes bfloat16, float16 and float32 tensors, not {bad[:3]}")
        dims = [self._block_dim(k, ls[0], dim) for k, (ls, _) in zip(keys, layers)]
        def shape(i):
            s = list(layers[i][0][0].shape)
            s[dims[i]] = len(ids[i]) if not isinstance(ids[i], torch.Tensor) else ids[i].numel()
            return [len(layers[i][0])] + s if layers[i][1] else s

        blocks, dev = [None] * len(keys), []
        for i, ((ls, _), d) in enumerate(zip(layers, dims)):
            # packed: the fused pack takes whole MX blocks under a fusable config, as put_blocks
            if ls[0].is_cuda and self._device_ids(ids[i], ls[0].device) and (
                    not pack_fp8 or (self._fusable_fp8_cfg(cfg) and self.client.device_fp8_eligible(torch.Size(shape(i)).numel()))):
                blocks[i] = self._device_blocks(ls, d, ids[i], None, 0, pack_fp8)
            if blocks[i] is not None:
                dev.append(i)
        rest = [i for i in range(len(keys)) if blocks[i] is None]
        refused = []
        if dev:
            ecs = {}
            if pack_fp8:  # one call per wide type
                for dt, grp in _by_dtype(dev, lambda i: layers[i][0][0].dtype).items():
                    got = self.client.batch_put_device_fp8_blocks([keys[i] for i in grp], [blocks[i][0] for i in grp], cfg, self._stream(),
                                                                  wide=_MX_WIDE[dt])
                    ecs.update(zip(grp, got))
            else:
                ecs.update(zip(dev, self.client.batch_put_device_blocks([keys[i] for i in dev], [blocks[i][0] for i in dev], cfg, self._stream())))
            ok = [i for i in dev if ecs[i] == _bb.ErrorCode.OK]
            rest += [i for i in dev if ecs[i] == _bb.ErrorCode.NOT_IMPLEMENTED]
            refused = [(i, ecs[i]) for i in dev if ecs[i] not in (_bb.ErrorCode.OK, _bb.ErrorCode.NOT_IMPLEMENTED)]
            if ok:
                self._put_metas([keys[i] for i in ok], [_meta(layers[i][0][0].dtype, shape(i), pack_fp8) for i in ok])
        if rest:
            sel = {i: torch.from_numpy(self._block_ids(keys[i], ids[i], layers[i][0][0].shape[dims[i]])) for i in rest}
            picked = []
            for i in rest:
                ls, stacked = layers[i]
                t = [c.index_select(dims[i], sel[i].to(c.device)) for c in ls]
                picked.append(torch.stack(t) if stacked else t[0])
            self.batch_put([keys[i] for i in rest], picked, pack_fp8, config)
        self._verdicts(keys, [i for i, _ in refused], [e for _, e in refused])

    def put_layer_blocks(self, key: str, caches, ids, dim: int = 0, pack_fp8: bool = False, config=None) -> None:
        """Stores `torch.stack([c.index_select(dim, ids) for c in caches])` under `key` (see batch_put_layer_blocks)."""
        self.batch_put_layer_blocks([key], [caches], [ids], dim, pack_fp8, config)

    def batch_get_layer_blocks_into(self, keys: Sequence[str], caches: Sequence, ids: Sequence, dim: int = 0,
                                    blocks: Optional[Sequence] = None) -> list:
        """The mirror of batch_put_layer_blocks: `c.index_copy_(dim, ids[i], stored[l])` for every layer l, c =
        caches[i][l], of the tensor stored under keys[i] (a single tensor: `caches[i].index_copy_(dim, ids[i], stored)`).
        With `blocks`, a partial restore: `stored[l].index_select(dim, blocks[i])` is copied instead.  Returns `caches`.

        Errors that need no ids come first, before any transfer: KeyError for a missing key, TypeError for a dtype other
        than the stored one, ValueError for a stored shape other than the selection's (with blocks: other than the
        caches' outside `dim`, or len(blocks[i]) != len(ids[i])) or for caches not on the current CUDA device.

        CUDA int32 or int64 `ids` (and `blocks`) on the caches' device stay there when every cache has the layout
        get_blocks_into stores into in place, with pages of at least LAYER_BLOCKS_MIN_PAGE_BYTES, and the layers do not
        overlap: the transfer engine builds the page table from them on the device (batch_get_device_blocks), with no host
        synchronisation.  A packed whole-block object takes batch_get_device_fp8_blocks (pages of at least
        FP8_LAYER_BLOCKS_MIN_PAGE_BYTES, one call per dtype), which unpacks each tile straight into its pages.  Then an id or block out of range (IndexError) or a repeated one (ValueError) is found on the
        device and raised after the call: no byte of that key's caches is written, and the other keys complete.  This
        differs from get_blocks_into, which checks before any transfer.  Every other case checks the ids on the host first
        (copying CUDA tensors there, which synchronises) and takes a whole get + index_copy_ per layer."""
        keys, caches, ids = list(keys), list(caches), list(ids)
        if not len(keys) == len(caches) == len(ids):
            raise ValueError("keys, caches and ids differ in length")
        if blocks is not None:
            blocks = list(blocks)
            if len(blocks) != len(keys):
                raise ValueError("keys and blocks differ in length")
        metas = self._metas(keys)
        dev = torch.cuda.current_device()
        layers = [self._layers(k, c) for k, c in zip(keys, caches)]
        dims = [self._block_dim(k, ls[0], dim) for k, (ls, _) in zip(keys, layers)]
        n_stored = []
        for j, (k, m, (ls, stacked), d) in enumerate(zip(keys, metas, layers, dims)):
            c = ls[0]
            if c.dtype != _stored_dtype(m):
                raise TypeError(f"{k}: cache is {c.dtype}, the stored tensor {_stored_dtype(m)}")
            if not c.is_cuda or c.device.index != dev:
                raise ValueError(f"{k}: caches must be CUDA tensors on cuda:{dev}, not {c.device}")
            stored = m["shape"][1:] if stacked else m["shape"]
            if stacked and (not m["shape"] or m["shape"][0] != len(ls)):
                raise ValueError(f"{k}: the stored tensor has shape {m['shape']}, for {len(ls)} layers")
            n = len(ids[j]) if not isinstance(ids[j], torch.Tensor) else ids[j].numel()
            if len(stored) != c.dim() or any(a != s for e, (a, s) in enumerate(zip(stored, c.shape)) if e != d):
                raise ValueError(f"{k}: the stored tensor has shape {m['shape']}, the caches {list(c.shape)}: they differ outside dim {d}")
            if blocks is None and stored[d] != n:
                raise ValueError(f"{k}: {stored[d]} blocks stored, {n} ids")
            if blocks is not None:
                nb = len(blocks[j]) if not isinstance(blocks[j], torch.Tensor) else blocks[j].numel()
                if nb != n:
                    raise ValueError(f"{k}: {nb} blocks for {n} ids")
            n_stored.append(stored[d])
        live = [i for i in range(len(keys)) if blocks is None or (len(blocks[i]) if not isinstance(blocks[i], torch.Tensor) else blocks[i].numel())]
        tables = [None] * len(keys)
        for i in live:
            ls = layers[i][0]
            sel = None if blocks is None else blocks[i]
            # packed objects the fused unpack reads (whole MX blocks) take the fp8 call; padded ones the fallback
            fp8 = metas[i]["packed"] is not None
            if (fp8 and not self._fp8_whole(metas[i])) or not self._device_ids(ids[i], ls[0].device) or (
                    sel is not None and not self._device_ids(sel, ls[0].device)):
                continue
            tables[i] = self._device_blocks(ls, dims[i], ids[i], sel, n_stored[i], fp8)
        on_dev = [i for i in live if tables[i] is not None and not metas[i]["packed"]]
        packed = [i for i in live if tables[i] is not None and metas[i]["packed"]]
        rest = [i for i in live if tables[i] is None]
        refused = []
        for dt, grp in _by_dtype(packed, lambda i: layers[i][0][0].dtype).items():  # one call per wide type
            ecs = self.client.batch_get_device_fp8_blocks([keys[i] for i in grp], [tables[i][0] for i in grp], self._stream(), wide=_MX_WIDE[dt])
            rest += [i for i, e in zip(grp, ecs) if e == _bb.ErrorCode.NOT_IMPLEMENTED]
            refused += [(i, e) for i, e in zip(grp, ecs) if e not in (_bb.ErrorCode.OK, _bb.ErrorCode.NOT_IMPLEMENTED)]
        if on_dev:
            ecs, sizes = self.client.batch_get_device_blocks([keys[i] for i in on_dev], [tables[i][0] for i in on_dev], self._stream())
            for i, e, n in zip(on_dev, ecs, sizes):
                want = int(np.prod(metas[i]["shape"], dtype=np.int64)) * layers[i][0][0].element_size()
                if e == _bb.ErrorCode.NOT_IMPLEMENTED:
                    rest.append(i)
                elif e == _bb.ErrorCode.OK and n != want:
                    raise RuntimeError(f"{keys[i]}: {n} bytes stored, {want} expected")
                elif e != _bb.ErrorCode.OK:
                    refused.append((i, e))
        if rest:
            idx, sel = {}, {}
            for i in rest:
                c = layers[i][0][0]
                idx[i] = self._block_ids(keys[i], ids[i], c.shape[dims[i]])
                if np.unique(idx[i]).size != idx[i].size:
                    raise ValueError(f"{keys[i]}: duplicate block ids")
                if blocks is not None:
                    sel[i] = self._block_ids(keys[i], blocks[i], n_stored[i], "blocks")
                    if np.unique(sel[i]).size != sel[i].size:
                        raise ValueError(f"{keys[i]}: duplicate blocks")

            def restore(i, t):
                ls, stacked = layers[i]
                for l, c in enumerate(ls):
                    s = t[l] if stacked else t
                    if i in sel:
                        s = s.index_select(dims[i], torch.from_numpy(sel[i]).to(s.device))
                    c.index_copy_(dims[i], torch.from_numpy(idx[i]).to(c.device), s)

            self._whole(keys, rest, None, restore)
        self._verdicts(keys, [i for i, _ in refused], [e for _, e in refused])
        return caches

    def get_layer_blocks_into(self, key: str, caches, ids, dim: int = 0, blocks=None):
        """The tensor stored under `key` copied into the blocks `ids` of every layer's cache (see
        batch_get_layer_blocks_into)."""
        return self.batch_get_layer_blocks_into([key], [caches], [ids], dim, None if blocks is None else [blocks])[0]

    # ------------------------------------------------------------------ get
    def _metas(self, keys: Sequence[str], bundle: bool = False) -> list:
        """The `#meta` records of keys: KeyError for a missing one, TypeError for a bundle where a tensor is wanted or the
        other way round (`bundle`)."""
        metas = []
        for k, (ec, blob) in zip(keys, self.client.batch_get([k + "#meta" for k in keys])):
            if ec != _bb.ErrorCode.OK:
                raise KeyError(f"object metadata missing: {ec}")
            m = json.loads(blob)
            if ("bundle" in m) != bundle:
                have, want = ("bundle", "tensor") if "bundle" in m else ("tensor", "bundle")
                raise TypeError(f"{k} holds a {have}, not a {want}: use the {want} calls")
            metas.append(m)
        return metas

    def batch_get(self, keys: Sequence[str], device: Optional[torch.device] = None) -> list:
        device = device or torch.device("cuda", torch.cuda.current_device())
        metas = self._metas(keys)
        keys = list(keys)
        result = [None] * len(keys)
        # MXFP8 objects made of whole tiles: unpack fused into the get kernel (falls through when the object is not a
        # single GPU-fabric shard any more, e.g. after demotion to a host tier)
        def call(grp, es, wide):
            for i in grp:
                result[i] = torch.empty(metas[i]["shape"], dtype=_stored_dtype(metas[i]), device=device)
            return self.client.batch_get_device_fp8([keys[i] for i in grp], [result[i].data_ptr() for i in grp],
                                                    [metas[i]["numel"] for i in grp], self._stream(), wide=wide)

        fused = [i for i, m in enumerate(metas) if self._fp8_whole(m)]
        for i in self._packed("fused fp8 get", keys, fused, lambda i: _stored_dtype(metas[i]), call):
            result[i] = None
        rest = [i for i in range(len(keys)) if result[i] is None]
        if not rest:
            return result
        all_keys, all_metas = keys, metas
        keys, metas = [all_keys[i] for i in rest], [all_metas[i] for i in rest]
        bufs = []
        for m in metas:
            if m["packed"] == "mxfp8":
                bufs.append(torch.empty(_bb.mxfp8_packed_bytes(m["padded_numel"]), dtype=torch.uint8, device=device))
            else:
                bufs.append(torch.empty(m["shape"], dtype=_DTYPES[m["dtype"]], device=device))
        ecs, sizes = self.client.batch_get_device(list(keys), [b.data_ptr() for b in bufs], [b.numel() * b.element_size() for b in bufs],
                                                  self._stream())
        _check("get", keys, ecs)
        out = []
        for m, b in zip(metas, bufs):
            if m["packed"] == "mxfp8":
                dt = _stored_dtype(m)  # unpacked straight to the stored dtype
                t = torch.empty(m["padded_numel"], dtype=dt, device=device)
                _bb.mxfp8_unpack(b.data_ptr(), m["padded_numel"], t.data_ptr(), self._stream(), wide=_MX_WIDE[dt])
                out.append(t[: m["numel"]].view(m["shape"]))
            else:
                out.append(b)
        for i, t in zip(rest, out):
            result[i] = t
        return result

    def get(self, key: str, device: Optional[torch.device] = None) -> torch.Tensor:
        return self.batch_get([key], device)[0]

    def batch_get_into(self, keys: Sequence[str], outs: Sequence[torch.Tensor]) -> list:
        """Loads each stored tensor into an existing CUDA tensor on the current device and returns `outs`: restoring a KV
        block into its slot of a preallocated cache (`cache[layer, :, slot]`), a tensor-parallel shard into its columns of
        a full weight (`W[:, k0:k1]`), or a tensor into a parameter's storage.  No element of an out's storage outside the
        view is written.  The outs must not overlap one another (not checked).

        Every check comes before any transfer: KeyError for a missing key, TypeError unless out.dtype is the stored
        dtype (packed tensors included), ValueError unless out.shape is the stored shape and out is a CUDA tensor on
        the current device.  Then each route is one call for all the tensors that take it:
          1. unpacked, contiguous out: batch_get_device into its storage;
          2. unpacked, out whose elements are rows (see _source_rows: `narrow` along any dim, `t[::k]`):
             batch_get_device_scatter, whose kernel stores each tile straight into the rows (misaligned rows are staged
             through the host by the client);
          3. MXFP8-packed whole-block tensors, contiguous or rows: batch_get_device_fp8, or batch_get_device_fp8_scatter
             when any out is rows (contiguous ones go as one row);
          4. everything else -- transposed or overlapping layouts, padded packed tensors, packed tensors the fused
             kernels refuse (NOT_IMPLEMENTED: misaligned rows, unfusable placements) -- batch_get into a temporary, then
             out.copy_()."""
        keys, outs = list(keys), list(outs)
        if len(keys) != len(outs):
            raise ValueError("keys and outs differ in length")
        metas = self._metas(keys)
        dev = torch.cuda.current_device()
        for k, m, o in zip(keys, metas, outs):
            want = _stored_dtype(m)
            if o.dtype != want:
                raise TypeError(f"{k}: out is {o.dtype}, the stored tensor {want}")
            if list(o.shape) != m["shape"]:
                raise ValueError(f"{k}: out has shape {list(o.shape)}, the stored tensor {m['shape']}")
            if not o.is_cuda or o.device.index != dev:
                raise ValueError(f"{k}: out must be a CUDA tensor on cuda:{dev}, not {o.device}")
        rows = [None if o.is_contiguous() else self._source_rows(o) for o in outs]
        plain = [i for i, m in enumerate(metas) if not m["packed"]]
        dense = [i for i in plain if outs[i].is_contiguous()]
        if dense:
            ecs, _ = self.client.batch_get_device([keys[i] for i in dense], [outs[i].data_ptr() for i in dense],
                                                  [outs[i].numel() * outs[i].element_size() for i in dense], self._stream())
            _check("get", [keys[i] for i in dense], ecs)
        scattered = [i for i in plain if rows[i] is not None]
        if scattered:
            ecs, _ = self.client.batch_get_device_scatter([keys[i] for i in scattered], [outs[i].data_ptr() for i in scattered],
                                                          [rows[i][0] for i in scattered], [rows[i][1] for i in scattered],
                                                          [rows[i][2] for i in scattered], self._stream())
            _check("scattered get", [keys[i] for i in scattered], ecs)
        rest = [i for i in plain if not outs[i].is_contiguous() and rows[i] is None]  # route 4
        packed = [i for i, m in enumerate(metas) if m["packed"]]
        fused = [i for i in packed if self._fp8_whole(metas[i]) and (outs[i].is_contiguous() or rows[i] is not None)]
        take = set(fused)
        rest += [i for i in packed if i not in take]

        def call(grp, es, wide):
            fk, ptrs, n = [keys[i] for i in grp], [outs[i].data_ptr() for i in grp], [outs[i].numel() for i in grp]
            if any(rows[i] is not None for i in grp):
                # contiguous outs go as one row each
                shapes = [_elem_rows(es, rows[i], outs[i].numel()) for i in grp]
                return self.client.batch_get_device_fp8_scatter(fk, ptrs, n, *map(list, zip(*shapes)), self._stream(), wide=wide)
            return self.client.batch_get_device_fp8(fk, ptrs, n, self._stream(), wide=wide)

        rest += self._packed("fused fp8 get", keys, fused, lambda i: outs[i].dtype, call)
        self._whole(keys, rest, None, lambda i, t: outs[i].copy_(t))
        return outs

    def get_into(self, key: str, out: torch.Tensor) -> torch.Tensor:
        """Loads the tensor stored under `key` into `out` and returns it (see batch_get_into)."""
        return self.batch_get_into([key], [out])[0]

    def batch_get_rows(self, keys: Sequence[str], starts: Sequence[int], stops: Sequence[int],
                       device: Optional[torch.device] = None) -> list:
        """Rows [start, stop) along dim 0 of each stored tensor, as new tensors (`t[start:stop]`): a tensor-parallel rank
        loads its shard of a weight, a reader a few KV blocks of a layer.  Only the byte range of those rows is stored
        into the result; every shard of the object that overlaps it is still read whole and verified against its
        digest.  IndexError unless 0 <= start <= stop <= shape[0]; 0-d tensors have no rows.  MXFP8-packed tensors take
        the fused element-range get: the whole packed object is read and verified, only the rows' elements are unpacked
        and stored.  Packed tensors the fused kernel cannot read (striped, demoted to a host tier) are read whole,
        unpacked and sliced."""
        device = device or torch.device("cuda", torch.cuda.current_device())
        keys, starts, stops = list(keys), list(starts), list(stops)
        if not len(keys) == len(starts) == len(stops):
            raise ValueError("keys, starts and stops differ in length")
        metas = self._metas(keys)
        for k, m, a, b in zip(keys, metas, starts, stops):
            if not m["shape"]:
                raise IndexError(f"{k}: a 0-d tensor has no rows")
            if not 0 <= a <= b <= m["shape"][0]:
                raise IndexError(f"{k}: rows [{a}, {b}) outside [0, {m['shape'][0]}]")
        return self._get_windows(keys, metas, [0] * len(keys), starts, stops, device)

    @staticmethod
    def _windows(metas: list, dims: list, starts: list, stops: list) -> list:
        """(offset, width, pitch, rows) of `t.narrow(dims[i], starts[i], stops[i] - starts[i])` of each stored tensor:
        `rows` = prod(shape[:dim]) runs of `width` units every `pitch` units from unit `offset`, the units elements for
        packed tensors, else bytes."""
        win = []
        for m, d, a, b in zip(metas, dims, starts, stops):
            shape = m["shape"]
            inner = torch.Size(shape[d + 1:]).numel()
            es = 1 if m["packed"] else _stored_dtype(m).itemsize
            win.append((a * inner * es, (b - a) * inner * es, shape[d] * inner * es, torch.Size(shape[:d]).numel()))
        return win

    def _get_windows(self, keys: list, metas: list, dims: list, starts: list, stops: list, device: torch.device) -> list:
        """`t.narrow(dims[i], starts[i], stops[i] - starts[i])` of each stored tensor, as new contiguous tensors.  The
        window is `rows` = prod(shape[:dim]) runs of `width` elements every `pitch` from element `offset`; the packed calls
        count elements, the others bytes.  Along dim 0 (one run) the range calls read it, along other dims the strided
        calls, one call per kind for all such items (packed: per dtype).  Packed items the fused kernel refuses are read
        whole and narrowed."""
        result, win = [None] * len(keys), self._windows(metas, dims, starts, stops)
        for i, (m, d, a, b) in enumerate(zip(metas, dims, starts, stops)):
            shape, dt = m["shape"], _stored_dtype(m)
            inner = torch.Size(shape[d + 1:]).numel()
            rows, offset, width = torch.Size(shape[:d]).numel(), a * inner, (b - a) * inner
            # Each result but an unpacked dim-0 one sits at element offset % (16 / element size) of its own allocation,
            # so that its virtual base (ptr - element size * offset) is 16-byte aligned and the window takes the fused
            # kernel whenever its row gap allows.
            skew = offset % (16 // dt.itemsize) if m["packed"] or d else 0
            result[i] = torch.empty(rows * width + skew, dtype=dt, device=device)[skew:].view(shape[:d] + [b - a] + shape[d + 1:])

        def narrowed(i, t):
            result[i] = t.narrow(dims[i], starts[i], stops[i] - starts[i]).clone(memory_format=torch.contiguous_format)

        for along0 in (True, False):
            idx = [i for i, d in enumerate(dims) if (d == 0) == along0]
            n = 2 if along0 else 4  # (offset, width) or (offset, width, pitch, rows)
            fp8_call, call, what = ((self.client.batch_get_device_fp8_range, self.client.batch_get_device_range, "range get") if along0 else
                                    (self.client.batch_get_device_fp8_strided, self.client.batch_get_device_strided, "strided get"))

            def fp8(grp, es, wide):
                return fp8_call([keys[i] for i in grp], [result[i].data_ptr() for i in grp], [metas[i]["padded_numel"] for i in grp],
                                *[[win[i][k] for i in grp] for k in range(n)], self._stream(), wide=wide)

            def dtype_of(i):
                return result[i].dtype

            # the items one dtype's call refuses are read whole before the next dtype's call
            for grp in _by_dtype([i for i in idx if metas[i]["packed"]], dtype_of).values():
                self._whole(keys, self._packed(f"fused fp8 {what}", keys, grp, dtype_of, fp8), device, narrowed)
            plain = [i for i in idx if not metas[i]["packed"]]
            if plain:
                ecs = call([keys[i] for i in plain], [result[i].data_ptr() for i in plain], *[[win[i][k] for i in plain] for k in range(n)],
                           self._stream())
                _check(what, [keys[i] for i in plain], ecs)
        return result

    def get_rows(self, key: str, start: int, stop: int, device: Optional[torch.device] = None) -> torch.Tensor:
        """`t[start:stop]` of the tensor stored under `key` (see batch_get_rows)."""
        return self.batch_get_rows([key], [start], [stop], device)[0]

    def batch_get_slices(self, keys: Sequence[str], dims: Sequence[int], starts: Sequence[int], stops: Sequence[int],
                         device: Optional[torch.device] = None) -> list:
        """`t.narrow(dim, start, stop - start).contiguous()` of each stored tensor, along any dimension: a row-parallel rank
        loads its columns `W[:, k0:k1]` of a weight stored whole, a decode rank its heads `kv[:, :, h0:h1, :]` of a KV
        layer.  Negative dims count from the end.  IndexError for 0-d tensors, a dim out of range, or bounds outside
        0 <= start <= stop <= shape[dim].

        dim 0 is batch_get_rows.  Along any other dim the slice is prod(shape[:dim]) rows of the same width, one per
        index of the outer dims, and the strided device get stores just those rows, densely: every shard of the object
        that holds a byte of them is read whole and verified against its digest, shards wholly between two rows are not
        read.  Each result starts at byte `offset % 16` of its own allocation, so that single-shard tensors take the fused
        kernel for every slice whose row gap is a multiple of 16 bytes; other slices are staged through the host.

        MXFP8-packed tensors, padded ones included (their pad lies past the last row), take the fused strided get of
        packed tensors: the whole packed object is read and verified against its digest, only the rows' elements are
        unpacked and stored.  Each result starts at element `offset % (16 / element size)` of its own allocation, so only a
        slice whose row gap is not a multiple of that many elements (8 for bf16 and fp16, 4 for fp32) misses the fused kernel; such slices, and packed tensors the fused kernel
        cannot read (striped, demoted to a host tier), are read whole, unpacked and narrowed."""
        device = device or torch.device("cuda", torch.cuda.current_device())
        keys, dims, starts, stops = list(keys), list(dims), list(starts), list(stops)
        if not len(keys) == len(dims) == len(starts) == len(stops):
            raise ValueError("keys, dims, starts and stops differ in length")
        metas = self._metas(keys)
        self._slice_checks(keys, metas, dims, starts, stops)
        return self._get_windows(keys, metas, dims, starts, stops, device)

    def get_slice(self, key: str, dim: int, start: int, stop: int, device: Optional[torch.device] = None) -> torch.Tensor:
        """`t.narrow(dim, start, stop - start).contiguous()` of the tensor stored under `key` (see batch_get_slices)."""
        return self.batch_get_slices([key], [dim], [start], [stop], device)[0]

    def _slice_checks(self, keys: list, metas: list, dims: list, starts: list, stops: list) -> None:
        """IndexError for a 0-d tensor, a dim out of range or bounds outside 0 <= start <= stop <= shape[dim]; dims are
        normalised in place (negative dims count from the end)."""
        for j, (k, m, a, b) in enumerate(zip(keys, metas, starts, stops)):
            shape = m["shape"]
            if not shape:
                raise IndexError(f"{k}: a 0-d tensor has no dimension to slice")
            if not -len(shape) <= dims[j] < len(shape):
                raise IndexError(f"{k}: dim {dims[j]} out of range for {len(shape)} dimensions")
            dims[j] %= len(shape)
            if not 0 <= a <= b <= shape[dims[j]]:
                raise IndexError(f"{k}: [{a}, {b}) outside [0, {shape[dims[j]]}] along dim {dims[j]}")

    def batch_get_slices_into(self, keys: Sequence[str], outs: Sequence[torch.Tensor], dims: Sequence[int], starts: Sequence[int],
                              stops: Sequence[int]) -> list:
        """Loads `t.narrow(dim, start, stop - start)` of each stored tensor into an existing CUDA tensor and returns `outs`:
        a tensor-parallel rank loads its shard of a stored weight into its place in a fused parameter
        (`W_fused[:, a:b]`), a reader restores heads `kv[:, h0:h1, :]` of a stored layer into the same heads of a live
        buffer, a job refreshes a slice of a model buffer in place.  No slice-sized temporary is made on the fused routes,
        and no element of an out's storage outside the view is written.  The outs must not overlap one another (not
        checked).

        Every check comes before any transfer: KeyError for a missing key; IndexError for a 0-d tensor, a dim out of
        range or bounds outside 0 <= start <= stop <= shape[dim] (negative dims count from the end); TypeError unless
        out.dtype is the stored dtype; ValueError unless out.shape is the narrowed shape and out is a CUDA tensor on the
        current device.  Then each route is one call for all the slices that take it (packed: one per dtype):
          1. a contiguous out: the range get (dim 0) or the strided get of batch_get_slices, at out's pointer;
          2. an out whose elements are rows (see _source_rows: `narrow` along any dim, `t[::k]`):
             batch_get_device_strided_scatter (packed: batch_get_device_fp8_strided_scatter), whose kernel stores the
             slice's pieces straight into the rows;
          3. everything else -- transposed or overlapping outs, and packed slices the fused kernels refuse
             (NOT_IMPLEMENTED: misaligned rows, unfusable placements) -- batch_get_slices into a temporary, then
             out.copy_().  Unpacked slices the fused kernels cannot store are staged through the host by the client."""
        keys, outs, dims, starts, stops = list(keys), list(outs), list(dims), list(starts), list(stops)
        if not len(keys) == len(outs) == len(dims) == len(starts) == len(stops):
            raise ValueError("keys, outs, dims, starts and stops differ in length")
        metas = self._metas(keys)
        self._slice_checks(keys, metas, dims, starts, stops)
        for k, m, o, d, a, b in zip(keys, metas, outs, dims, starts, stops):
            want = _stored_dtype(m)
            if o.dtype != want:
                raise TypeError(f"{k}: out is {o.dtype}, the stored tensor {want}")
            shape = m["shape"][:d] + [b - a] + m["shape"][d + 1:]
            if list(o.shape) != shape:
                raise ValueError(f"{k}: out has shape {list(o.shape)}, the slice {shape}")
            if not o.is_cuda or o.device.index != torch.cuda.current_device():
                raise ValueError(f"{k}: out must be a CUDA tensor on the current device, not {o.device}")
        win = self._windows(metas, dims, starts, stops)
        rows = [None if o.is_contiguous() else self._source_rows(o) for o in outs]
        n = len(keys)
        rest = [i for i in range(n) if not outs[i].is_contiguous() and rows[i] is None]  # route 3
        for along0 in (True, False):  # route 1: (offset, width) or (offset, width, pitch, rows) at out's pointer
            idx = [i for i in range(n) if outs[i].is_contiguous() and (dims[i] == 0) == along0]
            k = 2 if along0 else 4
            fp8_call, call, what = ((self.client.batch_get_device_fp8_range, self.client.batch_get_device_range, "range get") if along0 else
                                    (self.client.batch_get_device_fp8_strided, self.client.batch_get_device_strided, "strided get"))

            def fp8(grp, es, wide):
                return fp8_call([keys[i] for i in grp], [outs[i].data_ptr() for i in grp], [metas[i]["padded_numel"] for i in grp],
                                *[[win[i][j] for i in grp] for j in range(k)], self._stream(), wide=wide)

            rest += self._packed(f"fused fp8 {what}", keys, [i for i in idx if metas[i]["packed"]], lambda i: outs[i].dtype, fp8)
            plain = [i for i in idx if not metas[i]["packed"]]
            if plain:
                ecs = call([keys[i] for i in plain], [outs[i].data_ptr() for i in plain], *[[win[i][j] for i in plain] for j in range(k)],
                           self._stream())
                _check(what, [keys[i] for i in plain], ecs)
        idx = [i for i in range(n) if not outs[i].is_contiguous() and rows[i] is not None]  # route 2

        def dst_rows(grp, es):
            return [rows[i][0] // es for i in grp], [rows[i][1] // es for i in grp]

        def fp8_rows(grp, es, wide):
            return self.client.batch_get_device_fp8_strided_scatter(
                [keys[i] for i in grp], [outs[i].data_ptr() for i in grp], [metas[i]["padded_numel"] for i in grp],
                *[[win[i][j] for i in grp] for j in range(4)], *dst_rows(grp, es), self._stream(), wide=wide)

        rest += self._packed("fused fp8 slice get", keys, [i for i in idx if metas[i]["packed"]], lambda i: outs[i].dtype, fp8_rows)
        plain = [i for i in idx if not metas[i]["packed"]]
        if plain:
            ecs = self.client.batch_get_device_strided_scatter([keys[i] for i in plain], [outs[i].data_ptr() for i in plain],
                                                               *[[win[i][j] for i in plain] for j in range(4)], *dst_rows(plain, 1),
                                                               self._stream())
            _check("slice get", [keys[i] for i in plain], ecs)
        if rest:
            got = self._get_windows([keys[i] for i in rest], [metas[i] for i in rest], [dims[i] for i in rest], [starts[i] for i in rest],
                                    [stops[i] for i in rest], outs[rest[0]].device)
            for i, t in zip(rest, got):
                outs[i].copy_(t)
        return outs

    def get_slice_into(self, key: str, out: torch.Tensor, dim: int, start: int, stop: int) -> torch.Tensor:
        """Loads `t.narrow(dim, start, stop - start)` of the tensor stored under `key` into `out` and returns it (see
        batch_get_slices_into)."""
        return self.batch_get_slices_into([key], [out], [dim], [start], [stop])[0]

    def batch_get_rows_into(self, keys: Sequence[str], outs: Sequence[torch.Tensor], starts: Sequence[int], stops: Sequence[int]) -> list:
        """Rows [start, stop) along dim 0 of each stored tensor into existing tensors: batch_get_slices_into with dim 0."""
        keys = list(keys)
        return self.batch_get_slices_into(keys, outs, [0] * len(keys), starts, stops)

    def get_rows_into(self, key: str, out: torch.Tensor, start: int, stop: int) -> torch.Tensor:
        """`t[start:stop]` of the tensor stored under `key` into `out` (see batch_get_slices_into)."""
        return self.batch_get_slices_into([key], [out], [0], [start], [stop])[0]

    # ------------------------------------------------------------------ bundles
    def _gap_zeros(self, device: torch.device) -> torch.Tensor:
        """144 zero bytes at a 16-byte aligned address on `device`: the source of every gap between a bundle's tensors, and
        of a packed bundle's padding (up to 31 fp32 elements, 124 bytes, from an address up to 15 bytes in)."""
        cache = self.__dict__.setdefault("_gap_zero_bufs", {})
        if device not in cache:
            cache[device] = torch.zeros(144, dtype=torch.uint8, device=device)
        return cache[device]

    @staticmethod
    def _aligned(t: torch.Tensor, keep: list) -> torch.Tensor:
        """t itself when it is contiguous and 16-byte aligned (or has no elements), else an aligned contiguous copy kept
        alive in `keep`."""
        if t.numel() and (not t.is_contiguous() or t.data_ptr() % 16):
            t = t.clone(memory_format=torch.contiguous_format) if t.is_contiguous() else t.contiguous()
            if t.data_ptr() % 16:  # a fresh allocation is aligned; this is a guard, not a route
                t = torch.empty_like(t).copy_(t)
            keep.append(t)
        return t

    @staticmethod
    def _bundle_items(bundle, what: str) -> tuple:
        """(container kind, [(name, value)]) of a mapping (a state_dict) or a sequence, whose names are its indices."""
        if isinstance(bundle, dict) or hasattr(bundle, "items"):
            return "dict", [(str(k), v) for k, v in bundle.items()]
        if isinstance(bundle, (list, tuple)):
            return "list", [(str(i), v) for i, v in enumerate(bundle)]
        raise TypeError(f"{what}: a bundle is a mapping of names to tensors or a sequence of tensors, not {type(bundle).__name__}")

    def batch_put_bundles(self, keys: Sequence[str], bundles: Sequence, config=None, pack_fp8: bool = False) -> None:
        """Stores each bundle -- a mapping of names to CUDA tensors, such as a `state_dict`, or a sequence of them -- as
        ONE object under its key, with one `#meta`: the tensors back to back, each at a 16-byte aligned offset, read in
        place by the fused put kernel from a segment list (batch_put_device_segments), one native call for the batch.  A
        bundle costs one object's control-plane work instead of two per tensor, and it is stored whole or not at all.

        The gaps between tensors are read from a small zeroed device buffer at an address congruent to the gap's offset,
        so a bundle of 16-byte aligned contiguous tensors is read wholly in place; a tensor that is not contiguous or not
        16-byte aligned is copied into an aligned temporary first.  Every dtype TensorStore knows is accepted, 0-d and
        zero-element tensors included.  TypeError for another dtype or a value that is not a tensor, ValueError for a
        tensor that is not a CUDA tensor on the current device; both before anything is stored.  The `#meta` records
        each entry's name, dtype, shape, offset and bytes and the total.

        pack_fp8 stores each bundle as ONE MXFP8-packed object (see _put_packed_bundles): every entry of a bundle must
        have the same dtype, bf16, fp16 or fp32 (TypeError otherwise), and a bundle needs at least one element
        (ValueError), both before anything is stored."""
        cfg = config or self.config
        keys, bundles = list(keys), list(bundles)
        if len(keys) != len(bundles):
            raise ValueError("keys and bundles differ in length")
        plans = []
        for k, b in zip(keys, bundles):
            kind, items = self._bundle_items(b, k)
            dts = {t.dtype for _, t in items if isinstance(t, torch.Tensor)}
            if pack_fp8 and (len(dts) > 1 or not dts <= set(_MX_WIDE)):
                raise TypeError(f"{k}: a packed bundle holds bfloat16, float16 or float32 tensors of one dtype, not {sorted(map(str, dts))}")
            for name, t in items:
                if not isinstance(t, torch.Tensor):
                    raise TypeError(f"{k}[{name}]: not a tensor but {type(t).__name__}")
                if t.dtype not in _DTYPES.values():
                    raise TypeError(f"{k}[{name}]: dtype {t.dtype} is not one TensorStore stores")
                if not t.is_cuda or t.device.index != torch.cuda.current_device():
                    raise ValueError(f"{k}[{name}]: must be a CUDA tensor on the current device, not {t.device}")
            if pack_fp8 and sum(t.numel() for _, t in items) == 0:
                raise ValueError(f"{k}: a packed bundle needs at least one element")
            plans.append((kind, items))
        if pack_fp8:
            self._put_packed_bundles(keys, plans, cfg)
            return
        zeros = self._gap_zeros(torch.device("cuda", torch.cuda.current_device())).data_ptr()
        segments, metas, keep = [], [], []
        for kind, items in plans:
            segs, entries, off = [], [], 0
            for name, t in items:
                nbytes = t.numel() * t.element_size()
                t = self._aligned(t, keep)
                gap = -off % 16
                if gap:
                    segs.append((zeros + off % 16, gap))
                    off += gap
                if nbytes:
                    segs.append((t.data_ptr(), nbytes))
                entries.append({"name": name, "dtype": str(t.dtype).replace("torch.", ""), "shape": list(t.shape), "offset": off,
                                "bytes": nbytes})
                off += nbytes
            segments.append(np.array(segs, dtype=np.uint64).reshape(-1, 2))
            metas.append(json.dumps({"bundle": kind, "entries": entries, "total": off}).encode())
        ecs = self.client.batch_put_device_segments(keys, segments, cfg, self._stream())
        _check("bundle put", keys, ecs)
        self._put_metas(keys, metas)

    def _put_packed_bundles(self, keys: list, plans: list, cfg) -> None:
        """The packed form of batch_put_bundles, for checked (kind, items) plans.  Each entry starts on a whole 32-element
        MX block and is padded with zeros to a multiple of 32 elements, so its values never share a block scale with a
        neighbour's: each entry decodes bit for bit to what put(k, t, pack_fp8=True) and get(k) give for it alone.  The
        padding is read from the zeroed gap buffer at an address congruent to its wide-byte offset, and entries that are
        not contiguous or not 16-byte aligned get an aligned temporary, so the fused pack reads the segment list in place
        (batch_put_device_fp8_segments, one call per dtype) when the config is fusable.  Otherwise, and for bundles it
        refuses with NOT_IMPLEMENTED, the entries are copied into a padded wide temporary, packed (mxfp8_pack) and put as
        bytes: the stored object is byte for byte the same.  The `#meta` is the plain bundle's record, offsets and bytes in
        wide bytes of the unpacked object, plus "packed", "dtype" and "numel", the padded element total."""
        zeros = self._gap_zeros(torch.device("cuda", torch.cuda.current_device())).data_ptr()
        segments, metas, dtypes, numels, keep = [], [], [], [], []
        for kind, items in plans:
            dt = items[0][1].dtype
            es = dt.itemsize
            segs, entries, off = [], [], 0  # off in elements
            for name, t in items:
                n = t.numel()
                t = self._aligned(t, keep)
                if n:
                    segs.append((t.data_ptr(), n))
                entries.append({"name": name, "dtype": str(dt).replace("torch.", ""), "shape": list(t.shape), "offset": es * off,
                                "bytes": es * n})
                off += n
                pad = -off % 32
                if pad:
                    segs.append((zeros + es * off % 16, pad))
                    off += pad
            segments.append(np.array(segs, dtype=np.uint64).reshape(-1, 2))
            metas.append({"bundle": kind, "entries": entries, "total": es * off, "packed": "mxfp8",
                          "dtype": str(dt).replace("torch.", ""), "numel": off})
            dtypes.append(dt)
            numels.append(off)
        idx = list(range(len(keys)))
        if self._fusable_fp8_cfg(cfg):
            def call(grp, es, wide):
                return self.client.batch_put_device_fp8_segments([keys[i] for i in grp], [segments[i] for i in grp], cfg, self._stream(),
                                                                 wide=wide)

            idx = self._packed("packed bundle put", keys, idx, lambda i: dtypes[i], call)
        if idx:
            packed = []
            for i in idx:
                wide = torch.zeros(numels[i], dtype=dtypes[i], device=torch.device("cuda", torch.cuda.current_device()))
                for (_, t), e in zip(plans[i][1], metas[i]["entries"]):
                    if e["bytes"]:
                        self._entry_view(wide.view(torch.uint8), e).copy_(t)
                buf = torch.empty(_bb.mxfp8_packed_bytes(numels[i]), dtype=torch.uint8, device=wide.device)
                _bb.mxfp8_pack(wide.data_ptr(), numels[i], buf.data_ptr(), self._stream(), wide=_MX_WIDE[dtypes[i]])
                packed.append(buf)
            ecs = self.client.batch_put_device([keys[i] for i in idx], [b.data_ptr() for b in packed], [b.numel() for b in packed], cfg,
                                               self._stream())
            _check("packed bundle put", [keys[i] for i in idx], ecs)
        self._put_metas(keys, [json.dumps(m).encode() for m in metas])

    def put_bundle(self, key: str, tensors, config=None, pack_fp8: bool = False) -> None:
        """Stores the mapping or sequence of CUDA tensors `tensors` as one object (see batch_put_bundles)."""
        self.batch_put_bundles([key], [tensors], config, pack_fp8)

    @staticmethod
    def _entry_view(buf: torch.Tensor, e: dict) -> torch.Tensor:
        dt = _DTYPES[e["dtype"]]
        return buf[e["offset"]: e["offset"] + e["bytes"]].view(dt).view(e["shape"])

    def _packed_bundle_bufs(self, keys: list, metas: list, idx: list, bufs: list, device) -> None:
        """Fills bufs[i], for each packed bundle i of idx, with its unpacked object as bytes: one fused unpack per dtype
        (batch_get_device_fp8) into a wide allocation; a bundle it refuses with NOT_IMPLEMENTED is read packed
        (batch_get_device) and unpacked by mxfp8_unpack."""
        wides = {i: torch.empty(metas[i]["numel"], dtype=_stored_dtype(metas[i]), device=device) for i in idx}
        for i in idx:
            bufs[i] = wides[i].view(torch.uint8)

        def call(grp, es, wide):
            return self.client.batch_get_device_fp8([keys[i] for i in grp], [wides[i].data_ptr() for i in grp],
                                                    [metas[i]["numel"] for i in grp], self._stream(), wide=wide)

        rest = [i for i in idx if not self.client.device_fp8_eligible(metas[i]["numel"])]
        rest += self._packed("packed bundle get", keys, [i for i in idx if i not in rest], lambda i: _stored_dtype(metas[i]), call)
        if rest:
            packed = [torch.empty(_bb.mxfp8_packed_bytes(metas[i]["numel"]), dtype=torch.uint8, device=device) for i in rest]
            ecs, _ = self.client.batch_get_device([keys[i] for i in rest], [b.data_ptr() for b in packed], [b.numel() for b in packed],
                                                  self._stream())
            _check("packed bundle get", [keys[i] for i in rest], ecs)
            for i, b in zip(rest, packed):
                _bb.mxfp8_unpack(b.data_ptr(), metas[i]["numel"], wides[i].data_ptr(), self._stream(), wide=_MX_WIDE[_stored_dtype(metas[i])])

    def batch_get_bundles(self, keys: Sequence[str], device: Optional[torch.device] = None) -> list:
        """Each stored bundle in the container type it was stored as (a dict, or a list for a sequence), its tensors views
        of ONE aligned allocation per bundle that a single plain device get (batch_get_device) filled and verified: the
        views share that storage, so resizing one or keeping one alive keeps the whole bundle's allocation.  TypeError
        for a key that holds a tensor, KeyError for a missing one.  A packed bundle's allocation is its unpacked object,
        filled by one fused unpack per dtype (see _packed_bundle_bufs); a batch may mix packed and plain bundles."""
        device = device or torch.device("cuda", torch.cuda.current_device())
        keys = list(keys)
        metas = self._metas(keys, bundle=True)
        bufs = [torch.empty(max(m["total"], 1), dtype=torch.uint8, device=device) if not m.get("packed") else None for m in metas]
        self._packed_bundle_bufs(keys, metas, [i for i, m in enumerate(metas) if m.get("packed")], bufs, device)
        idx = [i for i, m in enumerate(metas) if m["total"] and not m.get("packed")]
        if idx:
            ecs, _ = self.client.batch_get_device([keys[i] for i in idx], [bufs[i].data_ptr() for i in idx], [metas[i]["total"] for i in idx],
                                                  self._stream())
            _check("bundle get", [keys[i] for i in idx], ecs)
        out = []
        for m, b in zip(metas, bufs):
            views = [(e["name"], self._entry_view(b, e)) for e in m["entries"]]
            out.append(dict(views) if m["bundle"] == "dict" else [v for _, v in views])
        return out

    def get_bundle(self, key: str, device: Optional[torch.device] = None):
        """The bundle stored under `key` (see batch_get_bundles)."""
        return self.batch_get_bundles([key], device)[0]

    def batch_get_bundles_into(self, keys: Sequence[str], outs: Sequence) -> list:
        """Loads stored bundles into existing CUDA tensors in place -- a checkpoint into a module's parameters -- and
        returns `outs`.  outs[i] maps entry names to tensors (a sequence stands for names 0, 1, ...) and may name a subset:
        the entries it does not name, and the gaps, are not stored.  Every bundle is one segment list of ONE
        batch_get_device_segments call: a contiguous 16-byte aligned out is a segment itself, any other out gets a
        contiguous temporary segment and then out.copy_(tmp).  Every shard of the object is still read whole and
        verified.  Packed bundles take one batch_get_device_fp8_segments call per dtype instead, their segments in
        elements (the padding is a null segment too); one it refuses with NOT_IMPLEMENTED is read whole (see
        _packed_bundle_bufs) and copied into the outs.  A batch may mix packed and plain bundles.

        Every check comes before any transfer: KeyError for a missing key or name, TypeError for a key that holds a
        tensor or an out of another dtype than its entry, ValueError for another shape or an out that is not a CUDA
        tensor on the current device."""
        keys, outs = list(keys), list(outs)
        if len(keys) != len(outs):
            raise ValueError("keys and outs differ in length")
        metas = self._metas(keys, bundle=True)
        dev = torch.cuda.current_device()
        named = []
        for k, m, o in zip(keys, metas, outs):
            _, items = self._bundle_items(o, k)
            entries = {e["name"]: e for e in m["entries"]}
            for name, t in items:
                if name not in entries:
                    raise KeyError(f"{k}: the bundle has no entry {name!r}")
                e = entries[name]
                if not isinstance(t, torch.Tensor):
                    raise TypeError(f"{k}[{name}]: not a tensor but {type(t).__name__}")
                if t.dtype != _DTYPES[e["dtype"]]:
                    raise TypeError(f"{k}[{name}]: out is {t.dtype}, the stored tensor {e['dtype']}")
                if list(t.shape) != e["shape"]:
                    raise ValueError(f"{k}[{name}]: out has shape {list(t.shape)}, the stored tensor {e['shape']}")
                if not t.is_cuda or t.device.index != dev:
                    raise ValueError(f"{k}[{name}]: out must be a CUDA tensor on cuda:{dev}, not {t.device}")
            named.append(dict(items))
        segments, copies = [], []
        for i, (m, want) in enumerate(zip(metas, named)):
            es = _stored_dtype(m).itemsize if m.get("packed") else 1  # segments in elements of a packed bundle
            segs, off = [], 0
            for e in m["entries"]:
                if e["offset"] > off:
                    segs.append((0, (e["offset"] - off) // es))
                t = want.get(e["name"])
                if e["bytes"] and t is None:
                    segs.append((0, e["bytes"] // es))
                elif e["bytes"]:
                    if not t.is_contiguous() or t.data_ptr() % 16:
                        tmp = torch.empty(e["shape"], dtype=t.dtype, device=t.device)
                        copies.append((i, t, tmp))
                        t = tmp
                    segs.append((t.data_ptr(), e["bytes"] // es))
                off = e["offset"] + e["bytes"]
            if m["total"] > off:  # a packed bundle's last padding
                segs.append((0, (m["total"] - off) // es))
            segments.append(np.array(segs, dtype=np.uint64).reshape(-1, 2))
        plain = [i for i, m in enumerate(metas) if not m.get("packed")]
        if plain:
            ecs, _ = self.client.batch_get_device_segments([keys[i] for i in plain], [segments[i] for i in plain], self._stream())
            _check("bundle get", [keys[i] for i in plain], ecs)

        def call(grp, es, wide):
            ecs, _ = self.client.batch_get_device_fp8_segments([keys[i] for i in grp], [segments[i] for i in grp], self._stream(), wide=wide)
            return ecs

        packed = [i for i, m in enumerate(metas) if m.get("packed")]
        rest = self._packed("packed bundle get", keys, packed, lambda i: _stored_dtype(metas[i]), call)
        for i, t, tmp in copies:
            if i not in rest:
                t.copy_(tmp)
        if rest:  # refused: the whole unpacked object, then each named entry copied out of it
            bufs = [None] * len(keys)
            self._packed_bundle_bufs(keys, metas, rest, bufs, torch.device("cuda", dev))
            for i in rest:
                for e in metas[i]["entries"]:
                    if e["name"] in named[i] and e["bytes"]:
                        named[i][e["name"]].copy_(self._entry_view(bufs[i], e))
        return outs

    def get_bundle_into(self, key: str, outs):
        """Loads the bundle stored under `key` into the tensors `outs` names (see batch_get_bundles_into)."""
        return self.batch_get_bundles_into([key], [outs])[0]

    def remove(self, keys: Sequence[str]) -> None:
        self.client.batch_remove(list(keys) + [k + "#meta" for k in keys])

    def keys(self, prefix: str = "", limit: int = 0) -> list:
        """Names of the tensors stored under `prefix` (key order; the `#meta` side objects are hidden)."""
        out, after = [], ""
        while True:
            page = self.client.keystone().list_objects(prefix, 1000, after)
            out += [k for k, _, _, _ in page if not k.endswith("#meta")]
            if len(page) < 1000 or (limit and len(out) >= limit):
                return out[:limit] if limit else out
            after = page[-1][0]


class AsyncTensorStore(TensorStore):
    """TensorStore whose puts / gets run on a side stream from a worker thread, so they overlap the caller's compute
    (KV-cache offload, activation checkpoints).  `put_async` orders itself after the work already queued on the
    caller's stream (event wait), returns a `concurrent.futures.Future`; `get_async`'s future yields the tensors, already
    synchronised with the side stream.  The native calls release the GIL."""

    def __init__(self, client, config=None, workers: int = 1):
        super().__init__(client, config)
        from concurrent.futures import ThreadPoolExecutor

        self._pool = ThreadPoolExecutor(max_workers=workers, thread_name_prefix="bb-async")
        self._device = torch.cuda.current_device()
        self._side = torch.cuda.Stream(device=self._device)

    def _stream(self) -> int:  # every native call of this store is issued on the side stream
        return self._side.cuda_stream

    def _on_side(self, after_caller: bool, fn, *args, result=None):
        """A future of fn(*args) run on the side stream from the worker thread, after the work already queued on the
        caller's stream when `after_caller`; it yields `result` (fn's own result when None) once the side stream is done."""
        ready = None
        if after_caller:
            ready = torch.cuda.Event()
            ready.record(torch.cuda.current_stream())

        def run():
            torch.cuda.set_device(self._device)
            if ready is not None:
                self._side.wait_event(ready)
            with torch.cuda.stream(self._side):
                out = fn(*args)
            self._side.synchronize()
            return out if result is None else result

        return self._pool.submit(run)

    def put_async(self, keys: Sequence[str], tensors: Sequence[torch.Tensor], pack_fp8: bool = False, config=None):
        tensors = list(tensors)  # keep them alive until the transfer is done
        return self._on_side(True, self.batch_put, keys, tensors, pack_fp8, config, result=len(tensors))

    def get_async(self, keys: Sequence[str]):
        return self._on_side(False, self.batch_get, keys)

    def get_into_async(self, keys: Sequence[str], outs: Sequence[torch.Tensor]):
        """batch_get_into on the side stream; the future yields `outs`, already synchronised with it.  The side stream
        first waits for the work already queued on the caller's stream, so the get does not overtake the caller's earlier
        reads or writes of the outs."""
        outs = list(outs)
        return self._on_side(True, self.batch_get_into, list(keys), outs, result=outs)

    def get_slices_into_async(self, keys: Sequence[str], outs: Sequence[torch.Tensor], dims: Sequence[int], starts: Sequence[int],
                              stops: Sequence[int]):
        """batch_get_slices_into on the side stream, ordered after the work already queued on the caller's stream; the
        future yields `outs`, already synchronised with the side stream, or raises the call's error."""
        outs = list(outs)
        return self._on_side(True, self.batch_get_slices_into, list(keys), outs, list(dims), list(starts), list(stops), result=outs)

    def put_blocks_async(self, keys: Sequence[str], caches: Sequence[torch.Tensor], ids: Sequence, dim: int = 0, pack_fp8: bool = False,
                         config=None):
        """batch_put_blocks on the side stream, ordered after the work already queued on the caller's stream; the future
        yields the number of objects stored."""
        keys = list(keys)
        return self._on_side(True, self.batch_put_blocks, keys, list(caches), list(ids), dim, pack_fp8, config, result=len(keys))

    def get_blocks_into_async(self, keys: Sequence[str], caches: Sequence[torch.Tensor], ids: Sequence, dim: int = 0,
                              blocks: Optional[Sequence] = None):
        """batch_get_blocks_into (with `blocks`, a partial restore) on the side stream, ordered after the work already
        queued on the caller's stream; the future yields `caches`, already synchronised with the side stream."""
        caches = list(caches)
        return self._on_side(True, self.batch_get_blocks_into, list(keys), caches, list(ids), dim,
                             None if blocks is None else list(blocks), result=caches)

    def put_layer_blocks_async(self, keys: Sequence[str], caches: Sequence, ids: Sequence, dim: int = 0, pack_fp8: bool = False,
                               config=None):
        """batch_put_layer_blocks on the side stream, ordered after the work already queued on the caller's stream (which
        may be writing the ids); the future yields the number of objects stored, or raises the call's error."""
        keys = list(keys)
        return self._on_side(True, self.batch_put_layer_blocks, keys, list(caches), list(ids), dim, pack_fp8, config, result=len(keys))

    def get_layer_blocks_into_async(self, keys: Sequence[str], caches: Sequence, ids: Sequence, dim: int = 0,
                                    blocks: Optional[Sequence] = None):
        """batch_get_layer_blocks_into on the side stream, ordered after the work already queued on the caller's stream;
        the future yields `caches`, already synchronised with the side stream."""
        caches = list(caches)
        return self._on_side(True, self.batch_get_layer_blocks_into, list(keys), caches, list(ids), dim,
                             None if blocks is None else list(blocks), result=caches)

    def put_bundles_async(self, keys: Sequence[str], bundles: Sequence, config=None, pack_fp8: bool = False):
        """batch_put_bundles on the side stream, ordered after the work already queued on the caller's stream; the future
        yields the number of bundles stored, or raises the call's error."""
        keys, bundles = list(keys), list(bundles)  # keep the tensors alive until the transfer is done
        return self._on_side(True, self.batch_put_bundles, keys, bundles, config, pack_fp8, result=len(keys))

    def get_bundles_into_async(self, keys: Sequence[str], outs: Sequence):
        """batch_get_bundles_into on the side stream, ordered after the work already queued on the caller's stream; the
        future yields `outs`, already synchronised with the side stream."""
        outs = list(outs)
        return self._on_side(True, self.batch_get_bundles_into, list(keys), outs, result=outs)

    def close(self):
        self._pool.shutdown(wait=True)
