"""Torch-facing API: put / get CUDA tensors through the object store with the fused kernels.

    store = TensorStore(cluster.client)
    store.batch_put(["act/0", "act/1"], [t0, t1])                  # BBH64 digest fused into the copy
    store.put("kv/layer3", kv_fp16, pack_fp8=True)                  # block-scaled MXFP8 on the wire / in the slab
    t = store.get("kv/layer3")                                      # verified + unpacked fp16 tensor

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


def _stored_dtype(m) -> torch.dtype:
    """The dtype a stored tensor is returned as: its own, packed or not (packed metas always record it)."""
    return _DTYPES[m["dtype"]]


def _by_dtype(idx, dtype_of) -> dict:
    """idx grouped by dtype_of(i), in order: one native call per wide type."""
    groups = {}
    for i in idx:
        groups.setdefault(dtype_of(i), []).append(i)
    return groups


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

    # ------------------------------------------------------------------ put
    def _fused_fp8_ok(self, t: torch.Tensor, cfg) -> bool:
        """Pack fused into the put kernel: bf16, fp16 or fp32, a whole number of 32-element MX blocks, up to 3 copies (one
        tile pass fans out to every replica), each copy in one shard."""
        return (t.dtype in _MX_WIDE and self.client.device_fp8_eligible(t.numel()) and 1 <= cfg.replication_factor <= 3
                and cfg.max_workers_per_copy == 1 and t.data_ptr() % 16 == 0)

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
        if pack_fp8:
            # objects the fused kernel can take go through batch_put_device_fp8 (bf16 read once, packed bytes on the
            # wire, digest of the packed object from the tensor cores); the rest are packed first (unfused path below)
            fused_all = [i for i, t in enumerate(tensors) if t.is_cuda and self._fused_fp8_ok(t, cfg)]
            done = []
            for dt, fused in _by_dtype(fused_all, lambda i: tensors[i].dtype).items():
                fk = [keys[i] for i in fused]
                ptrs = [tensors[i].data_ptr() for i in fused]
                es, wide = tensors[fused[0]].element_size(), _MX_WIDE[dt]
                if any(rows[i] is not None for i in fused):
                    # one call and one launch: contiguous tensors go as one row each; widths and pitches in elements
                    shapes = [(rows[i][0] // es, rows[i][1] // es, rows[i][2]) if rows[i] is not None else (tensors[i].numel(),) * 2 + (1,)
                              for i in fused]
                    ecs = self.client.batch_put_device_fp8_strided(fk, ptrs, [s[0] for s in shapes], [s[1] for s in shapes],
                                                                   [s[2] for s in shapes], cfg, self._stream(), wide=wide)
                else:
                    ecs = self.client.batch_put_device_fp8(fk, ptrs, [tensors[i].numel() for i in fused], cfg, self._stream(), wide=wide)
                done += [i for i, e in zip(fused, ecs) if e == _bb.ErrorCode.OK]
                bad = [(keys[i], e) for i, e in zip(fused, ecs) if e not in (_bb.ErrorCode.OK, _bb.ErrorCode.NOT_IMPLEMENTED)]
                if bad:
                    raise RuntimeError(f"fused fp8 put failed: {bad[:3]}")
            if fused_all:
                metas = []
                for i in done:
                    t = tensors[i]
                    metas.append(json.dumps({"dtype": str(t.dtype).replace("torch.", ""), "shape": list(t.shape), "packed": "mxfp8",
                                             "numel": t.numel(), "padded_numel": t.numel()}).encode())
                if done:
                    ecs = self.client.batch_put([keys[i] + "#meta" for i in done], metas, self._meta_cfg())
                    if any(e != _bb.ErrorCode.OK for e in ecs):
                        raise RuntimeError("meta put failed")
                rest = [i for i in range(len(keys)) if i not in set(done)]
                # a gathered slice the fused put refused (its placement is not one GPU-fabric shard per copy) is made
                # contiguous and packed first, like any other
                keys, tensors = [keys[i] for i in rest], [tensors[i].contiguous() for i in rest]
                rows = [None] * len(keys)
                if not keys:
                    return
        payloads, metas, keep = [], [], []
        for t in tensors:
            assert t.is_cuda, "TensorStore moves CUDA tensors (host data: use client.put)"
            meta = {"dtype": str(t.dtype).replace("torch.", ""), "shape": list(t.shape), "packed": None, "numel": t.numel()}
            if pack_fp8:
                n = t.numel()
                npad = (n + 31) // 32 * 32
                src = t.view(-1)
                if npad != n:
                    src = torch.cat([src, torch.zeros(npad - n, dtype=t.dtype, device=t.device)])
                packed = torch.empty(_bb.mxfp8_packed_bytes(npad), dtype=torch.uint8, device=t.device)
                _bb.mxfp8_pack(src.data_ptr(), npad, packed.data_ptr(), self._stream(), wide=_MX_WIDE[t.dtype])
                keep.append(src)
                meta["packed"] = "mxfp8"
                meta["padded_numel"] = npad
                t = packed
            assert t.data_ptr() % 16 == 0, "tensor storage must be 16-byte aligned"
            payloads.append(t)
            metas.append(json.dumps(meta).encode())
        ptrs, sizes = [p.data_ptr() for p in payloads], [p.numel() * p.element_size() for p in payloads]
        if any(r is not None for r in rows):
            # one call and one launch for the whole batch: the other tensors go as one row each (pack_fp8 has no rows)
            shapes = [r if r is not None else (n, n, 1) for r, n in zip(rows, sizes)]
            ecs = self.client.batch_put_device_strided(list(keys), ptrs, [s[0] for s in shapes], [s[1] for s in shapes],
                                                       [s[2] for s in shapes], cfg, self._stream())
        else:
            ecs = self.client.batch_put_device(list(keys), ptrs, sizes, cfg, self._stream())
        bad = [(k, e) for k, e in zip(keys, ecs) if e != _bb.ErrorCode.OK]
        if bad:
            raise RuntimeError(f"put failed: {bad[:3]}")
        ecs = self.client.batch_put([k + "#meta" for k in keys], metas, self._meta_cfg())
        if any(e != _bb.ErrorCode.OK for e in ecs):
            raise RuntimeError("meta put failed")

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
    def _block_ids(key: str, ids, size: int) -> np.ndarray:
        """`ids` (a list or an integer tensor) as a 1-D int64 numpy array; a CUDA tensor is copied to the host once, which
        synchronises with its stream.  IndexError for an id outside [0, size)."""
        if isinstance(ids, torch.Tensor):
            if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
                raise TypeError(f"{key}: ids must be a 1-D integer list or tensor")
            a = ids.to(device="cpu", dtype=torch.int64).numpy()
        else:
            a = np.asarray(list(ids))
            if a.size == 0:
                a = a.astype(np.int64)
            if a.dtype.kind not in "iu":
                raise TypeError(f"{key}: ids must be a 1-D integer list or tensor")
            a = a.astype(np.int64)
        if a.ndim != 1:
            raise TypeError(f"{key}: ids must be a 1-D integer list or tensor")
        if a.size and (a.min() < 0 or a.max() >= size):
            raise IndexError(f"{key}: block ids must lie in [0, {size})")
        return a

    @staticmethod
    def _block_pages(cache: torch.Tensor, dim: int, ids: np.ndarray):
        """(page addresses, page bytes) of cache.index_select(dim, ids) for the paged device calls, or None when they should
        not move it.  Page (o, k) is cache[o..., ids[k]] over the dims after `dim`, in index_select order (outer index
        major): those dims must form one contiguous block of a multiple of 16 bytes, the outer dims must collapse to one
        positive stride, the blocks must not overlap one another (no zero or negative strides: an expanded cache takes
        the fallback), every page must be 16-byte aligned, and the page at least PAGED_MIN_PAGE_BYTES.  The addresses are a
        numpy int64 array, built without a loop per page."""
        if not cache.is_cuda or cache.numel() == 0 or ids.size == 0:
            return None
        es, shape, stride = cache.element_size(), cache.shape, cache.stride()
        page = es
        for n, s in reversed([(n, s) for n, s in zip(shape[dim + 1:], stride[dim + 1:]) if n != 1]):
            if s * es != page:
                return None
            page *= n
        if page % 16 or page < PAGED_MIN_PAGE_BYTES:
            return None
        outer = [(n, s) for n, s in zip(shape[:dim], stride[:dim]) if n != 1]
        if any(s != s2 * n2 for (_, s), (n2, s2) in zip(outer, outer[1:])):
            return None
        n_outer = int(np.prod([n for n, _ in outer], dtype=np.int64))
        o_step = outer[-1][1] * es if outer else 0
        b_step = stride[dim] * es
        # disjoint blocks: every (outer, block) step positive and at least the extent of the smaller steps' blocks
        extent = page
        for n, step in sorted([(n, st) for n, st in ((n_outer, o_step), (shape[dim], b_step)) if n > 1], key=lambda t: t[1]):
            if step < extent:
                return None
            extent = step * (n - 1) + extent
        addrs = (cache.data_ptr() + np.arange(n_outer, dtype=np.int64)[:, None] * o_step + ids[None, :] * b_step).reshape(-1)
        if (addrs & 15).any():
            return None
        return addrs, page

    def batch_put_blocks(self, keys: Sequence[str], caches: Sequence[torch.Tensor], ids: Sequence, dim: int = 0, pack_fp8: bool = False,
                         config=None) -> None:
        """Stores `caches[i].index_select(dim, ids[i])` under keys[i], with the usual `#meta`, so get, get_into, get_rows
        and get_slice read it unchanged: the blocks of a request in a paged KV cache, all layers at once, as one object.
        IndexError for an id out of range, before anything is stored.

        When the cache is a CUDA tensor whose dims after `dim` form one contiguous block of a multiple of 16 bytes and at
        least PAGED_MIN_PAGE_BYTES (32 KiB, where the paged calls start to beat index_select), whose outer dims collapse
        to one stride, whose blocks do not overlap and whose pages are 16-byte aligned, the blocks are read in place by
        the paged put (batch_put_device_paged): no index_select temporary, no extra device pass.  Any other layout, and
        pack_fp8, takes index_select and batch_put.  IndexError for a dim out of range.  A CUDA `ids` tensor is copied to the host once, which synchronises."""
        keys, caches, ids = list(keys), list(caches), list(ids)
        if not len(keys) == len(caches) == len(ids):
            raise ValueError("keys, caches and ids differ in length")
        dims = [self._block_dim(k, c, dim) for k, c in zip(keys, caches)]
        idx = [self._block_ids(k, b, c.shape[d]) for k, c, b, d in zip(keys, caches, ids, dims)]
        pages = [None if pack_fp8 else self._block_pages(c, d, b) for c, d, b in zip(caches, dims, idx)]
        paged = [i for i, p in enumerate(pages) if p is not None]
        if paged:
            ecs = self.client.batch_put_device_paged([keys[i] for i in paged], [pages[i][0] for i in paged], [pages[i][1] for i in paged],
                                                     config or self.config, self._stream())
            bad = [(keys[i], e) for i, e in zip(paged, ecs) if e != _bb.ErrorCode.OK]
            if bad:
                raise RuntimeError(f"paged put failed: {bad[:3]}")
            metas = []
            for i in paged:
                shape = list(caches[i].shape)
                shape[dims[i]] = idx[i].size
                metas.append(json.dumps({"dtype": str(caches[i].dtype).replace("torch.", ""), "shape": shape, "packed": None,
                                         "numel": torch.Size(shape).numel()}).encode())
            ecs = self.client.batch_put([keys[i] + "#meta" for i in paged], metas, self._meta_cfg())
            if any(e != _bb.ErrorCode.OK for e in ecs):
                raise RuntimeError("meta put failed")
        rest = [i for i, p in enumerate(pages) if p is None]
        if rest:
            self.batch_put([keys[i] for i in rest], [caches[i].index_select(dims[i], torch.from_numpy(idx[i]).to(caches[i].device)) for i in rest],
                           pack_fp8, config)

    def put_blocks(self, key: str, cache: torch.Tensor, ids, dim: int = 0, pack_fp8: bool = False, config=None) -> None:
        """Stores `cache.index_select(dim, ids)` under `key` (see batch_put_blocks)."""
        self.batch_put_blocks([key], [cache], [ids], dim, pack_fp8, config)

    def batch_get_blocks_into(self, keys: Sequence[str], caches: Sequence[torch.Tensor], ids: Sequence, dim: int = 0) -> list:
        """`caches[i].index_copy_(dim, ids[i], stored)` for the tensor stored under keys[i]: restores a request's KV blocks
        into whatever free blocks the allocator handed out.  No element of a cache outside the selected blocks is written.
        Returns `caches`.

        Every check comes before any transfer: KeyError for a missing key, TypeError unless the cache dtype is the stored
        dtype, ValueError unless the stored shape is the index_select shape, for a cache that is not a CUDA tensor on the
        current device and for duplicate ids, IndexError for an id or a dim out of range.  Caches of the layout
        batch_put_blocks reads in place take the paged get (batch_get_device_paged), which stores each tile straight into
        its pages (RuntimeError unless the stored object fills every selected block);
        other layouts, and packed tensors, take a get followed by index_copy_.  A CUDA `ids` tensor is copied to the host
        once, which synchronises."""
        keys, caches, ids = list(keys), list(caches), list(ids)
        if not len(keys) == len(caches) == len(ids):
            raise ValueError("keys, caches and ids differ in length")
        metas = self._metas(keys)
        dev = torch.cuda.current_device()
        dims = [self._block_dim(k, c, dim) for k, c in zip(keys, caches)]
        idx = []
        for k, m, c, b, d in zip(keys, metas, caches, ids, dims):
            if c.dtype != _stored_dtype(m):
                raise TypeError(f"{k}: cache is {c.dtype}, the stored tensor {_stored_dtype(m)}")
            t = self._block_ids(k, b, c.shape[d])
            shape = list(c.shape)
            shape[d] = t.size
            if shape != m["shape"]:
                raise ValueError(f"{k}: the stored tensor has shape {m['shape']}, the selected blocks {shape}")
            if not c.is_cuda or c.device.index != dev:
                raise ValueError(f"{k}: cache must be a CUDA tensor on cuda:{dev}, not {c.device}")
            if np.unique(t).size != t.size:
                raise ValueError(f"{k}: duplicate block ids")
            idx.append(t)
        pages = [None if m["packed"] else self._block_pages(c, d, b) for m, c, d, b in zip(metas, caches, dims, idx)]
        paged = [i for i, p in enumerate(pages) if p is not None]
        if paged:
            ecs, sizes = self.client.batch_get_device_paged([keys[i] for i in paged], [pages[i][0] for i in paged],
                                                            [pages[i][1] for i in paged], self._stream())
            bad = [(keys[i], e) for i, e in zip(paged, ecs) if e != _bb.ErrorCode.OK]
            # the stored object must fill every page: a shorter one would leave the last blocks as they were
            bad += [(keys[i], f"{n} bytes stored, {pages[i][0].size * pages[i][1]} selected") for i, e, n in zip(paged, ecs, sizes)
                    if e == _bb.ErrorCode.OK and n != pages[i][0].size * pages[i][1]]
            if bad:
                raise RuntimeError(f"paged get failed: {bad[:3]}")
        rest = [i for i, p in enumerate(pages) if p is None]
        if rest:
            for i, t in zip(rest, self.batch_get([keys[i] for i in rest], caches[rest[0]].device)):
                caches[i].index_copy_(dims[i], torch.from_numpy(idx[i]).to(caches[i].device), t)
        return caches

    def get_blocks_into(self, key: str, cache: torch.Tensor, ids, dim: int = 0) -> torch.Tensor:
        """`cache.index_copy_(dim, ids, stored)` for the tensor stored under `key` (see batch_get_blocks_into)."""
        return self.batch_get_blocks_into([key], [cache], [ids], dim)[0]

    # ------------------------------------------------------------------ get
    def _metas(self, keys: Sequence[str]) -> list:
        metas = []
        for ec, blob in self.client.batch_get([k + "#meta" for k in keys]):
            if ec != _bb.ErrorCode.OK:
                raise KeyError(f"object metadata missing: {ec}")
            metas.append(json.loads(blob))
        return metas

    def batch_get(self, keys: Sequence[str], device: Optional[torch.device] = None) -> list:
        device = device or torch.device("cuda", torch.cuda.current_device())
        metas = self._metas(keys)
        keys = list(keys)
        result = [None] * len(keys)
        # MXFP8 objects made of whole tiles: unpack fused into the get kernel (falls through when the object is not a
        # single GPU-fabric shard any more, e.g. after demotion to a host tier)
        fused_all = [i for i, m in enumerate(metas) if m["packed"] == "mxfp8" and m["padded_numel"] == m["numel"]
                     and self.client.device_fp8_eligible(m["numel"])]
        for dt, fused in _by_dtype(fused_all, lambda i: _stored_dtype(metas[i])).items():
            outs = [torch.empty(metas[i]["numel"], dtype=dt, device=device) for i in fused]
            ecs = self.client.batch_get_device_fp8([keys[i] for i in fused], [o.data_ptr() for o in outs], [metas[i]["numel"] for i in fused],
                                                   self._stream(), wide=_MX_WIDE[dt])
            for i, o, e in zip(fused, outs, ecs):
                if e == _bb.ErrorCode.OK:
                    result[i] = o.view(metas[i]["shape"])
                elif e != _bb.ErrorCode.NOT_IMPLEMENTED:
                    raise RuntimeError(f"fused fp8 get failed: {keys[i]}: {e}")
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
        bad = [(k, e) for k, e in zip(keys, ecs) if e != _bb.ErrorCode.OK]
        if bad:
            raise RuntimeError(f"get failed: {bad[:3]}")
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
        rest = []  # route 4

        def check(name, idx, ecs):
            bad = [(keys[i], e) for i, e in zip(idx, ecs) if e != _bb.ErrorCode.OK]
            if bad:
                raise RuntimeError(f"{name} failed: {bad[:3]}")

        plain = [i for i, m in enumerate(metas) if not m["packed"]]
        dense = [i for i in plain if outs[i].is_contiguous()]
        if dense:
            ecs, _ = self.client.batch_get_device([keys[i] for i in dense], [outs[i].data_ptr() for i in dense],
                                                  [outs[i].numel() * outs[i].element_size() for i in dense], self._stream())
            check("get", dense, ecs)
        scattered = [i for i in plain if not outs[i].is_contiguous() and rows[i] is not None]
        if scattered:
            ecs, _ = self.client.batch_get_device_scatter([keys[i] for i in scattered], [outs[i].data_ptr() for i in scattered],
                                                          [rows[i][0] for i in scattered], [rows[i][1] for i in scattered],
                                                          [rows[i][2] for i in scattered], self._stream())
            check("scattered get", scattered, ecs)
        rest += [i for i in plain if not outs[i].is_contiguous() and rows[i] is None]
        packed = [i for i, m in enumerate(metas) if m["packed"]]
        fused = [i for i in packed if metas[i]["padded_numel"] == metas[i]["numel"] and self.client.device_fp8_eligible(metas[i]["numel"])
                 and (outs[i].is_contiguous() or rows[i] is not None)]
        rest += [i for i in packed if i not in set(fused)]
        for dt, fused in _by_dtype(fused, lambda i: outs[i].dtype).items():
            fk, ptrs = [keys[i] for i in fused], [outs[i].data_ptr() for i in fused]
            es, wide = outs[fused[0]].element_size(), _MX_WIDE[dt]
            if any(rows[i] is not None for i in fused):
                # widths and pitches in elements; contiguous outs go as one row each
                shapes = [(rows[i][0] // es, rows[i][1] // es, rows[i][2]) if rows[i] is not None else (outs[i].numel(),) * 2 + (1,)
                          for i in fused]
                ecs = self.client.batch_get_device_fp8_scatter(fk, ptrs, [outs[i].numel() for i in fused], [s[0] for s in shapes],
                                                               [s[1] for s in shapes], [s[2] for s in shapes], self._stream(), wide=wide)
            else:
                ecs = self.client.batch_get_device_fp8(fk, ptrs, [outs[i].numel() for i in fused], self._stream(), wide=wide)
            check("fused fp8 get", [i for i, e in zip(fused, ecs) if e != _bb.ErrorCode.NOT_IMPLEMENTED],
                  [e for e in ecs if e != _bb.ErrorCode.NOT_IMPLEMENTED])
            rest += [i for i, e in zip(fused, ecs) if e == _bb.ErrorCode.NOT_IMPLEMENTED]
        if rest:
            for i, t in zip(rest, self.batch_get([keys[i] for i in rest], outs[rest[0]].device)):
                outs[i].copy_(t)
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
        return self._get_rows(keys, metas, starts, stops, device)

    def _get_rows(self, keys: list, metas: list, starts: list, stops: list, device: torch.device) -> list:
        result = [None] * len(keys)
        packed_all = [i for i, m in enumerate(metas) if m["packed"]]
        for dt, packed in _by_dtype(packed_all, lambda i: _stored_dtype(metas[i])).items():
            # Elements [lo, hi) of the (padded) packed object; their window ends before any pad.  Each result sits at
            # element lo % (16 / element size) of its own allocation, so that the virtual base ptr - size * lo is 16-byte
            # aligned and every row size takes the fused path.
            per = 16 // torch.empty((), dtype=dt).element_size()
            los, counts, ptrs = [], [], []
            for i in packed:
                m = metas[i]
                row = torch.Size(m["shape"][1:]).numel()
                lo, count = starts[i] * row, (stops[i] - starts[i]) * row
                buf = torch.empty(count + lo % per, dtype=dt, device=device)
                result[i] = buf[lo % per:].view([stops[i] - starts[i]] + m["shape"][1:])
                los.append(lo), counts.append(count), ptrs.append(result[i].data_ptr())
            ecs = self.client.batch_get_device_fp8_range([keys[i] for i in packed], ptrs, [metas[i]["padded_numel"] for i in packed], los,
                                                         counts, self._stream(), wide=_MX_WIDE[dt])
            bad = [(keys[i], e) for i, e in zip(packed, ecs) if e not in (_bb.ErrorCode.OK, _bb.ErrorCode.NOT_IMPLEMENTED)]
            if bad:
                raise RuntimeError(f"fused fp8 range get failed: {bad[:3]}")
            unfused = [i for i, e in zip(packed, ecs) if e == _bb.ErrorCode.NOT_IMPLEMENTED]
            if unfused:
                whole = self.batch_get([keys[i] for i in unfused], device)
                for i, t in zip(unfused, whole):
                    result[i] = t[starts[i]:stops[i]].clone()
        ranged = [i for i, m in enumerate(metas) if not m["packed"]]
        if ranged:
            offsets, lengths = [], []
            for i in ranged:
                m = metas[i]
                dtype = _DTYPES[m["dtype"]]
                row = torch.Size(m["shape"][1:]).numel() * torch.empty((), dtype=dtype).element_size()
                result[i] = torch.empty([stops[i] - starts[i]] + m["shape"][1:], dtype=dtype, device=device)
                offsets.append(starts[i] * row)
                lengths.append((stops[i] - starts[i]) * row)
            ecs = self.client.batch_get_device_range([keys[i] for i in ranged], [result[i].data_ptr() for i in ranged], offsets,
                                                     lengths, self._stream())
            bad = [(keys[i], e) for i, e in zip(ranged, ecs) if e != _bb.ErrorCode.OK]
            if bad:
                raise RuntimeError(f"range get failed: {bad[:3]}")
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
        for j, (k, m, a, b) in enumerate(zip(keys, metas, starts, stops)):
            shape = m["shape"]
            if not shape:
                raise IndexError(f"{k}: a 0-d tensor has no dimension to slice")
            if not -len(shape) <= dims[j] < len(shape):
                raise IndexError(f"{k}: dim {dims[j]} out of range for {len(shape)} dimensions")
            dims[j] %= len(shape)
            if not 0 <= a <= b <= shape[dims[j]]:
                raise IndexError(f"{k}: [{a}, {b}) outside [0, {shape[dims[j]]}] along dim {dims[j]}")
        result = [None] * len(keys)
        first = [i for i, d in enumerate(dims) if d == 0]
        if first:
            rows = self._get_rows([keys[i] for i in first], [metas[i] for i in first], [starts[i] for i in first],
                                  [stops[i] for i in first], device)
            for i, t in zip(first, rows):
                result[i] = t
        packed_all = [i for i, m in enumerate(metas) if dims[i] != 0 and m["packed"]]
        for dt, packed in _by_dtype(packed_all, lambda i: _stored_dtype(metas[i])).items():
            # prod(shape[:dim]) rows of (stop - start) * inner elements every shape[dim] * inner elements
            per = 16 // torch.empty((), dtype=dt).element_size()
            offsets, widths, pitches, nrows = [], [], [], []
            for i in packed:
                shape, d = metas[i]["shape"], dims[i]
                inner = torch.Size(shape[d + 1:]).numel()
                offset, width = starts[i] * inner, (stops[i] - starts[i]) * inner
                rows = torch.Size(shape[:d]).numel()
                buf = torch.empty(rows * width + offset % per, dtype=dt, device=device)
                result[i] = buf[offset % per:].view(shape[:d] + [stops[i] - starts[i]] + shape[d + 1:])
                offsets.append(offset), widths.append(width), pitches.append(shape[d] * inner), nrows.append(rows)
            ecs = self.client.batch_get_device_fp8_strided([keys[i] for i in packed], [result[i].data_ptr() for i in packed],
                                                           [metas[i]["padded_numel"] for i in packed], offsets, widths, pitches,
                                                           nrows, self._stream(), wide=_MX_WIDE[dt])
            bad = [(keys[i], e) for i, e in zip(packed, ecs) if e not in (_bb.ErrorCode.OK, _bb.ErrorCode.NOT_IMPLEMENTED)]
            if bad:
                raise RuntimeError(f"fused fp8 strided get failed: {bad[:3]}")
            unfused = [i for i, e in zip(packed, ecs) if e == _bb.ErrorCode.NOT_IMPLEMENTED]
            if unfused:
                for i, t in zip(unfused, self.batch_get([keys[i] for i in unfused], device)):
                    result[i] = t.narrow(dims[i], starts[i], stops[i] - starts[i]).contiguous()
        strided = [i for i, m in enumerate(metas) if dims[i] != 0 and not m["packed"]]
        if strided:
            offsets, widths, pitches, nrows = [], [], [], []
            for i in strided:
                shape, d, dtype = metas[i]["shape"], dims[i], _DTYPES[metas[i]["dtype"]]
                inner = torch.Size(shape[d + 1:]).numel() * torch.empty((), dtype=dtype).element_size()
                offset, width = starts[i] * inner, (stops[i] - starts[i]) * inner
                rows = torch.Size(shape[:d]).numel()
                buf = torch.empty(rows * width + offset % 16, dtype=torch.uint8, device=device)
                result[i] = buf[offset % 16:].view(dtype).view(shape[:d] + [stops[i] - starts[i]] + shape[d + 1:])
                offsets.append(offset), widths.append(width), pitches.append(shape[d] * inner), nrows.append(rows)
            ecs = self.client.batch_get_device_strided([keys[i] for i in strided], [result[i].data_ptr() for i in strided], offsets,
                                                       widths, pitches, nrows, self._stream())
            bad = [(keys[i], e) for i, e in zip(strided, ecs) if e != _bb.ErrorCode.OK]
            if bad:
                raise RuntimeError(f"strided get failed: {bad[:3]}")
        return result

    def get_slice(self, key: str, dim: int, start: int, stop: int, device: Optional[torch.device] = None) -> torch.Tensor:
        """`t.narrow(dim, start, stop - start).contiguous()` of the tensor stored under `key` (see batch_get_slices)."""
        return self.batch_get_slices([key], [dim], [start], [stop], device)[0]

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

    def put_async(self, keys: Sequence[str], tensors: Sequence[torch.Tensor], pack_fp8: bool = False, config=None):
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream())  # the tensors' producers
        tensors = list(tensors)  # keep them alive until the transfer is done

        def run():
            torch.cuda.set_device(self._device)
            self._side.wait_event(ready)
            with torch.cuda.stream(self._side):
                self.batch_put(keys, tensors, pack_fp8, config)
            self._side.synchronize()
            return len(tensors)

        return self._pool.submit(run)

    def get_async(self, keys: Sequence[str]):
        def run():
            torch.cuda.set_device(self._device)
            with torch.cuda.stream(self._side):
                out = self.batch_get(keys)
            self._side.synchronize()
            return out

        return self._pool.submit(run)

    def get_into_async(self, keys: Sequence[str], outs: Sequence[torch.Tensor]):
        """batch_get_into on the side stream; the future yields `outs`, already synchronised with it.  The side stream
        first waits for the work already queued on the caller's stream, so the get does not overtake the caller's earlier
        reads or writes of the outs."""
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream())
        keys, outs = list(keys), list(outs)

        def run():
            torch.cuda.set_device(self._device)
            self._side.wait_event(ready)
            with torch.cuda.stream(self._side):
                self.batch_get_into(keys, outs)
            self._side.synchronize()
            return outs

        return self._pool.submit(run)

    def put_blocks_async(self, keys: Sequence[str], caches: Sequence[torch.Tensor], ids: Sequence, dim: int = 0, pack_fp8: bool = False,
                         config=None):
        """batch_put_blocks on the side stream, ordered after the work already queued on the caller's stream; the future
        yields the number of objects stored."""
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream())
        keys, caches, ids = list(keys), list(caches), list(ids)

        def run():
            torch.cuda.set_device(self._device)
            self._side.wait_event(ready)
            with torch.cuda.stream(self._side):
                self.batch_put_blocks(keys, caches, ids, dim, pack_fp8, config)
            self._side.synchronize()
            return len(keys)

        return self._pool.submit(run)

    def get_blocks_into_async(self, keys: Sequence[str], caches: Sequence[torch.Tensor], ids: Sequence, dim: int = 0):
        """batch_get_blocks_into on the side stream, ordered after the work already queued on the caller's stream; the
        future yields `caches`, already synchronised with the side stream."""
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream())
        keys, caches, ids = list(keys), list(caches), list(ids)

        def run():
            torch.cuda.set_device(self._device)
            self._side.wait_event(ready)
            with torch.cuda.stream(self._side):
                self.batch_get_blocks_into(keys, caches, ids, dim)
            self._side.synchronize()
            return caches

        return self._pool.submit(run)

    def close(self):
        self._pool.shutdown(wait=True)
