"""Which native client calls each TensorStore method makes.  A recorder around the real client logs every `batch_*` call
with its address-free arguments (keys, sizes, widths, pitches, rows, page counts and page offsets, element counts,
`wide`, the `#meta` records byte for byte) and the error codes it returned, and forwards everything unchanged.  A fixed
table of cases reaches every route and every fallback: contiguous, row-view and transposed puts, packed and unpacked;
a mixed bf16 + fp16 + fp32 packed batch; blocks above and below each page threshold; get_into contiguous, row-view and
transposed outs; padded packed tensors; rows and slices along every dim; packed objects the fused kernels refuse with
NOT_IMPLEMENTED (an XXH3 digest, or read through misaligned rows).  A refused fused put needs a placement that is not
one GPU-fabric shard per copy, which one GPU cannot make.  Each case asserts the literal call list and every
result against a torch reference (an exact MXFP8 model for packed tensors)."""
import numpy as np
import pytest
import torch

from test_mxfp8_exhaustive import model_pack, model_unpack
from test_mxfp8_wide import model_pack_w, model_unpack_w

pytestmark = pytest.mark.gpu

IDS = [5, 0, 11]


def _entry(name, args, kw, res):
    """(name, address-free arguments..., error codes) of one client call."""
    out = [name]
    for j, a in enumerate(args):
        if hasattr(a, "replication_factor"):
            out.append(["cfg", a.replication_factor, a.max_workers_per_copy])
        elif isinstance(a, int):
            continue  # the stream
        elif j == 1 and "_device" in name:  # device addresses: page counts and offsets from the first page
            if "paged" in name:
                out.append([[int(x - p[0]) for x in p] for p in a])
        else:
            out.append([x.decode() if isinstance(x, bytes) else x if isinstance(x, str) else int(x) for x in a])
    if "wide" in kw:
        out.append(str(kw["wide"]))
    if name == "batch_get":
        res = [ec for ec, _ in res]
    out.append([str(e) for e in res[0]] + [list(res[1])] if isinstance(res, tuple) else [str(e) for e in res])
    return out


class Recorder:
    """The real client, with every batch_* call logged by _entry and forwarded unchanged."""

    def __init__(self, client):
        self.client, self.log = client, []

    def __getattr__(self, name):
        fn = getattr(self.client, name)
        if not name.startswith("batch_"):
            return fn

        def call(*args, **kw):
            res = fn(*args, **kw)
            self.log.append(_entry(name, args, kw, res))
            return res

        return call


def _bits(t):
    t = t.contiguous()
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _model(t):
    """unpack(pack(t)) by the exact MXFP8 model, in t's dtype and shape (padded to whole blocks for the model)."""
    x = _bits(t).cpu().numpy().reshape(-1)
    x = x.view({2: np.uint16, 4: np.uint32}[x.itemsize])
    n = x.size
    xp = np.concatenate([x, np.zeros(-n % 32, dtype=x.dtype)])
    if t.dtype == torch.bfloat16:
        y = model_unpack(model_pack(xp), xp.size)
    else:
        w = {torch.float16: "f16", torch.float32: "f32"}[t.dtype]
        y = model_unpack_w(model_pack_w(xp, w), xp.size, w)
    y = np.asarray(y)[:n].astype(x.dtype).view({2: np.int16, 4: np.int32}[x.itemsize])
    return torch.from_numpy(y.copy()).cuda().view(t.dtype).view(t.shape)


@pytest.fixture(scope="module")
def env():
    from blackbird_b200 import _bb
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")
    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-routes", dram_bytes=64 << 20)
    try:
        g = torch.Generator(device="cuda").manual_seed(11)

        def rnd(*shape, dtype=torch.bfloat16):
            return torch.randn(*shape, device="cuda", generator=g).to(dtype)

        D = {"W": rnd(256, 512), "H": rnd(64, 128, dtype=torch.float16), "F": rnd(32, 96, dtype=torch.float32),
             "kv": rnd(4, 2, 16, 64), "pad": rnd(7, 9), "X": rnd(50, 64),
             "cache": rnd(2, 16, 16, 8, 128), "small": rnd(2, 16, 4, 8, 128),                 # 32 KiB and 8 KiB pages
             "cache8": rnd(2, 16, 8, 8, 128), "small8": rnd(2, 16, 2, 8, 128),                # 16 KiB and 4 KiB pages
             "cache32": rnd(2, 16, 4, 8, 128, dtype=torch.float32),                          # 16 KiB pages
             # unfusable (packed first, then put); the fused unpack refuses the stored object, whose digest is not BBH64
             "xxh": _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, preferred_classes=[_bb.StorageClass.RAM_GPU],
                                     checksum=_bb.ChecksumAlgo.XXH3)}
        sel = {c: D[c].index_select(1, torch.tensor(IDS, device="cuda")) for c in ("cache", "small", "cache8", "small8", "cache32")}
        plain = TensorStore(cl.client)
        ref = {}
        for k, t, packed, cfg in [("w", D["W"], False, None), ("w8", D["W"], True, None), ("h8", D["H"], True, None),
                                  ("f8", D["F"], True, None), ("kv", D["kv"], False, None), ("kv8", D["kv"], True, None),
                                  ("pad8", D["pad"], True, None), ("x8s", D["X"], True, D["xxh"]), ("f8s", D["F"], True, D["xxh"]),
                                  ("blk", sel["cache"], False, None), ("sblk", sel["small"], False, None),
                                  ("blk8", sel["cache8"], True, None), ("sblk8", sel["small8"], True, None),
                                  ("blk32", sel["cache32"], True, None), ("blk8x", sel["cache8"], True, D["xxh"])]:
            plain.put(k, t, pack_fp8=packed, config=cfg)
            ref[k] = _model(t) if packed else t.clone()
        rec = Recorder(cl.client)
        yield cl, plain, TensorStore(rec), rec, D, ref
    finally:
        cl.stop()


def _puts(keys, tensors, packed=False, cfg=None):
    def run(store, plain, D, ref):
        ts = [t(D) for t in tensors]
        store.batch_put(keys, ts, pack_fp8=packed, config=cfg(D) if cfg else None)
        return [(plain.get(k), _model(t) if packed else t.contiguous()) for k, t in zip(keys, ts)]
    return run


def _put_blocks(keys, caches, packed=False, cfg=None):
    def run(store, plain, D, ref):
        store.batch_put_blocks(keys, [D[c] for c in caches], [IDS] * len(keys), dim=1, pack_fp8=packed, config=cfg(D) if cfg else None)
        want = [D[c].index_select(1, torch.tensor(IDS, device="cuda")) for c in caches]
        return [(plain.get(k), _model(w) if packed else w) for k, w in zip(keys, want)]
    return run


def _get_blocks_into(keys, caches):
    def run(store, plain, D, ref):
        outs = [torch.full_like(D[c], 3) for c in caches]
        ids = [[1, 9, 4]] * len(keys)
        got = store.batch_get_blocks_into(keys, outs, ids, dim=1)
        assert all(a is b for a, b in zip(got, outs))
        return [(o, torch.full_like(D[c], 3).index_copy_(1, torch.tensor(i, device="cuda"), ref[k]))
                for o, c, i, k in zip(outs, caches, ids, keys)]
    return run


def _get(keys):
    def run(store, plain, D, ref):
        return list(zip(store.batch_get(keys), [ref[k] for k in keys]))
    return run


def _get_into(keys, shapes, views):
    """views[i](base) is the out of keys[i] in a fresh base of shapes[i]; no element outside it may change."""
    def run(store, plain, D, ref):
        bases = [torch.full(s, 7, dtype=ref[k].dtype, device="cuda") for k, s in zip(keys, shapes)]
        outs = [v(b) for v, b in zip(views, bases)]
        got = store.batch_get_into(keys, outs)
        assert all(a is b for a, b in zip(got, outs))
        wants = [torch.full_like(b, 7) for b in bases]
        for k, v, w in zip(keys, views, wants):
            v(w).copy_(ref[k])
        return list(zip(bases, wants))
    return run


def _slices(items):
    """items: (key, dim, start, stop), all along dim 0 for get_rows; the results' 16-byte phases are logged too."""
    def run(store, plain, D, ref):
        keys, dims, starts, stops = map(list, zip(*items))
        if all(d == 0 for d in dims):
            got = store.batch_get_rows(keys, starts, stops)
        else:
            got = store.batch_get_slices(keys, dims, starts, stops)
        store.client.log.append(["phases", [o.data_ptr() % 16 for o in got]])
        return [(o, ref[k].narrow(d, a, b - a).contiguous()) for o, (k, d, a, b) in zip(got, items)]
    return run


CASES = {
    "put_contiguous": _puts(["p/c"], [lambda D: D["W"]]),
    "put_rows": _puts(["p/r"], [lambda D: D["W"][:, 128:256]]),
    "put_transposed": _puts(["p/t"], [lambda D: D["W"][:64, :32].t()]),
    "put_mixed": _puts(["p/m0", "p/m1", "p/m2"], [lambda D: D["W"], lambda D: D["kv"][:, :, 4:12, :], lambda D: D["W"][:64, :32].t()]),
    "put8_contiguous": _puts(["p8/c"], [lambda D: D["W"]], True),
    "put8_rows": _puts(["p8/r"], [lambda D: D["W"][:, 64:320]], True),
    "put8_transposed": _puts(["p8/t"], [lambda D: D["W"][:64, :64].t()], True),
    "put8_dtypes": _puts(["p8/b", "p8/h", "p8/f", "p8/pad", "p8/hr"],
                         [lambda D: D["W"], lambda D: D["H"], lambda D: D["F"], lambda D: D["pad"], lambda D: D["H"][:, 32:96]], True),
    "put8_unfusable": _puts(["p8/s0", "p8/s1"], [lambda D: D["X"], lambda D: D["W"][:, 64:320]], True, lambda D: D["xxh"]),
    "put_blocks": _put_blocks(["b/big", "b/small"], ["cache", "small"]),
    "put_blocks8": _put_blocks(["b8/big", "b8/small", "b8/f32", "b8/big2"], ["cache8", "small8", "cache32", "cache8"], True),
    "put_blocks8_unfusable": _put_blocks(["b8/x"], ["cache8"], True, lambda D: D["xxh"]),
    "get_blocks_into": _get_blocks_into(["blk", "sblk", "blk8", "sblk8", "blk32", "blk8x"],
                                        ["cache", "small", "cache8", "small8", "cache32", "cache8"]),
    "get": _get(["w", "w8", "h8", "f8", "pad8", "x8s", "f8s", "kv"]),
    # contiguous, rows, transposed (unpacked); contiguous, rows, misaligned rows, fp16, padded, refused rows and whole (packed)
    "get_into": _get_into(["w", "kv", "w", "w8", "w8", "w8", "h8", "pad8", "x8s", "x8s"],
                          [(256, 512), (4, 2, 32, 64), (512, 256), (256, 512), (256, 1024), (256, 1024), (64, 128), (7, 9),
                           (50, 128), (50, 64)],
                          [lambda B: B, lambda B: B[:, :, 8:24, :], lambda B: B.t(), lambda B: B, lambda B: B[:, 64:576],
                           lambda B: B[:, 3:515], lambda B: B, lambda B: B, lambda B: B[:, 64:128], lambda B: B]),
    "rows": _slices([("w", 0, 10, 50), ("w8", 0, 10, 50), ("f8", 0, 3, 30), ("pad8", 0, 2, 5), ("x8s", 0, 4, 9),
                     ("x8s", 0, 0, 50), ("f8s", 0, 3, 30), ("kv", 0, 1, 3), ("w", 0, 7, 7)]),
    "slices": _slices([("kv", 0, 1, 3), ("kv", 1, 1, 2), ("kv", 2, 3, 11), ("kv", -1, 5, 37), ("kv8", 1, 0, 1), ("kv8", 2, 8, 16),
                       ("kv8", 3, 3, 40), ("w8", 1, 3, 60), ("w", 1, 3, 60), ("pad8", 1, 1, 5), ("h8", 1, 32, 96),
                       ("f8", -1, 4, 20), ("x8s", 1, 8, 24), ("x8s", 1, 0, 32), ("f8s", 1, 4, 20), ("f8s", 0, 1, 2),
                       ("kv8", 0, 2, 4)]),
}

# the calls each case makes, in order: (name, address-free arguments..., error codes)
EXPECTED = {
    'put_contiguous': [['batch_put_device', ['p/c'], [262144], ['cfg', 1, 1], ['ErrorCode.OK']],
     ['batch_put', ['p/c#meta'], ['{"dtype": "bfloat16", "shape": [256, 512], "packed": null, "numel": 131072}'], ['cfg', 1, 1],
      ['ErrorCode.OK']]],
    'put_rows': [['batch_put_device_strided', ['p/r'], [256], [1024], [256], ['cfg', 1, 1], ['ErrorCode.OK']],
     ['batch_put', ['p/r#meta'], ['{"dtype": "bfloat16", "shape": [256, 128], "packed": null, "numel": 32768}'], ['cfg', 1, 1],
      ['ErrorCode.OK']]],
    'put_transposed': [['batch_put_device', ['p/t'], [4096], ['cfg', 1, 1], ['ErrorCode.OK']],
     ['batch_put', ['p/t#meta'], ['{"dtype": "bfloat16", "shape": [32, 64], "packed": null, "numel": 2048}'], ['cfg', 1, 1],
      ['ErrorCode.OK']]],
    'put_mixed': [['batch_put_device_strided', ['p/m0', 'p/m1', 'p/m2'], [262144, 1024, 4096], [262144, 2048, 4096], [1, 8, 1],
      ['cfg', 1, 1], ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_put', ['p/m0#meta', 'p/m1#meta', 'p/m2#meta'],
      ['{"dtype": "bfloat16", "shape": [256, 512], "packed": null, "numel": 131072}',
       '{"dtype": "bfloat16", "shape": [4, 2, 8, 64], "packed": null, "numel": 4096}',
       '{"dtype": "bfloat16", "shape": [32, 64], "packed": null, "numel": 2048}'],
      ['cfg', 1, 1], ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']]],
    'put8_contiguous': [['batch_put_device_fp8', ['p8/c'], [131072], ['cfg', 1, 1], 'MxWide.BF16', ['ErrorCode.OK']],
     ['batch_put', ['p8/c#meta'],
      ['{"dtype": "bfloat16", "shape": [256, 512], "packed": "mxfp8", "numel": 131072, "padded_numel": 131072}'], ['cfg', 1, 1],
      ['ErrorCode.OK']]],
    'put8_rows': [['batch_put_device_fp8_strided', ['p8/r'], [256], [512], [256], ['cfg', 1, 1], 'MxWide.BF16', ['ErrorCode.OK']],
     ['batch_put', ['p8/r#meta'],
      ['{"dtype": "bfloat16", "shape": [256, 256], "packed": "mxfp8", "numel": 65536, "padded_numel": 65536}'], ['cfg', 1, 1],
      ['ErrorCode.OK']]],
    'put8_transposed': [['batch_put_device_fp8', ['p8/t'], [4096], ['cfg', 1, 1], 'MxWide.BF16', ['ErrorCode.OK']],
     ['batch_put', ['p8/t#meta'],
      ['{"dtype": "bfloat16", "shape": [64, 64], "packed": "mxfp8", "numel": 4096, "padded_numel": 4096}'], ['cfg', 1, 1],
      ['ErrorCode.OK']]],
    'put8_dtypes': [['batch_put_device_fp8', ['p8/b'], [131072], ['cfg', 1, 1], 'MxWide.BF16', ['ErrorCode.OK']],
     ['batch_put_device_fp8_strided', ['p8/h', 'p8/hr'], [8192, 64], [8192, 128], [1, 64], ['cfg', 1, 1], 'MxWide.F16',
      ['ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_put_device_fp8', ['p8/f'], [3072], ['cfg', 1, 1], 'MxWide.F32', ['ErrorCode.OK']],
     ['batch_put', ['p8/b#meta', 'p8/h#meta', 'p8/hr#meta', 'p8/f#meta'],
      ['{"dtype": "bfloat16", "shape": [256, 512], "packed": "mxfp8", "numel": 131072, "padded_numel": 131072}',
       '{"dtype": "float16", "shape": [64, 128], "packed": "mxfp8", "numel": 8192, "padded_numel": 8192}',
       '{"dtype": "float16", "shape": [64, 64], "packed": "mxfp8", "numel": 4096, "padded_numel": 4096}',
       '{"dtype": "float32", "shape": [32, 96], "packed": "mxfp8", "numel": 3072, "padded_numel": 3072}'],
      ['cfg', 1, 1], ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_put_device', ['p8/pad'], [66], ['cfg', 1, 1], ['ErrorCode.OK']],
     ['batch_put', ['p8/pad#meta'],
      ['{"dtype": "bfloat16", "shape": [7, 9], "packed": "mxfp8", "numel": 63, "padded_numel": 64}'], ['cfg', 1, 1],
      ['ErrorCode.OK']]],
    'put8_unfusable': [['batch_put_device', ['p8/s0', 'p8/s1'], [3300, 67584], ['cfg', 1, 2], ['ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_put', ['p8/s0#meta', 'p8/s1#meta'],
      ['{"dtype": "bfloat16", "shape": [50, 64], "packed": "mxfp8", "numel": 3200, "padded_numel": 3200}',
       '{"dtype": "bfloat16", "shape": [256, 256], "packed": "mxfp8", "numel": 65536, "padded_numel": 65536}'],
      ['cfg', 1, 1], ['ErrorCode.OK', 'ErrorCode.OK']]],
    'put_blocks': [['batch_put_device_paged', ['b/big'], [[0, -163840, 196608, 524288, 360448, 720896]], [32768], ['cfg', 1, 1],
      ['ErrorCode.OK']],
     ['batch_put', ['b/big#meta'], ['{"dtype": "bfloat16", "shape": [2, 3, 16, 8, 128], "packed": null, "numel": 98304}'],
      ['cfg', 1, 1], ['ErrorCode.OK']],
     ['batch_put_device', ['b/small'], [49152], ['cfg', 1, 1], ['ErrorCode.OK']],
     ['batch_put', ['b/small#meta'], ['{"dtype": "bfloat16", "shape": [2, 3, 4, 8, 128], "packed": null, "numel": 24576}'],
      ['cfg', 1, 1], ['ErrorCode.OK']]],
    'put_blocks8': [['batch_put_device_fp8_paged', ['b8/big', 'b8/big2'],
      [[0, -81920, 98304, 262144, 180224, 360448], [0, -81920, 98304, 262144, 180224, 360448]], [8192, 8192], ['cfg', 1, 1],
      'MxWide.BF16', ['ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_put_device_fp8_paged', ['b8/f32'], [[0, -81920, 98304, 262144, 180224, 360448]], [4096], ['cfg', 1, 1],
      'MxWide.F32', ['ErrorCode.OK']],
     ['batch_put', ['b8/big#meta', 'b8/big2#meta', 'b8/f32#meta'],
      ['{"dtype": "bfloat16", "shape": [2, 3, 8, 8, 128], "packed": "mxfp8", "numel": 49152, "padded_numel": 49152}',
       '{"dtype": "bfloat16", "shape": [2, 3, 8, 8, 128], "packed": "mxfp8", "numel": 49152, "padded_numel": 49152}',
       '{"dtype": "float32", "shape": [2, 3, 4, 8, 128], "packed": "mxfp8", "numel": 24576, "padded_numel": 24576}'],
      ['cfg', 1, 1], ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_put_device_fp8', ['b8/small'], [12288], ['cfg', 1, 1], 'MxWide.BF16', ['ErrorCode.OK']],
     ['batch_put', ['b8/small#meta'],
      ['{"dtype": "bfloat16", "shape": [2, 3, 2, 8, 128], "packed": "mxfp8", "numel": 12288, "padded_numel": 12288}'],
      ['cfg', 1, 1], ['ErrorCode.OK']]],
    'put_blocks8_unfusable': [['batch_put_device', ['b8/x'], [50688], ['cfg', 1, 2], ['ErrorCode.OK']],
     ['batch_put', ['b8/x#meta'],
      ['{"dtype": "bfloat16", "shape": [2, 3, 8, 8, 128], "packed": "mxfp8", "numel": 49152, "padded_numel": 49152}'],
      ['cfg', 1, 1], ['ErrorCode.OK']]],
    'get_blocks_into': [['batch_get', ['blk#meta', 'sblk#meta', 'blk8#meta', 'sblk8#meta', 'blk32#meta', 'blk8x#meta'],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_get_device_fp8_paged', ['blk8', 'blk8x'],
      [[0, 131072, 49152, 262144, 393216, 311296], [0, 131072, 49152, 262144, 393216, 311296]], [8192, 8192], 'MxWide.BF16',
      ['ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device_fp8_paged', ['blk32'], [[0, 131072, 49152, 262144, 393216, 311296]], [4096], 'MxWide.F32',
      ['ErrorCode.OK']],
     ['batch_get_device_paged', ['blk'], [[0, 262144, 98304, 524288, 786432, 622592]], [32768], ['ErrorCode.OK', [196608]]],
     ['batch_get', ['sblk#meta', 'sblk8#meta', 'blk8x#meta'], ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_get_device_fp8', ['sblk8', 'blk8x'], [12288, 49152], 'MxWide.BF16', ['ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device', ['sblk', 'blk8x'], [49152, 50688], ['ErrorCode.OK', 'ErrorCode.OK', [49152, 50688]]]],
    'get': [['batch_get', ['w#meta', 'w8#meta', 'h8#meta', 'f8#meta', 'pad8#meta', 'x8s#meta', 'f8s#meta', 'kv#meta'],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK',
       'ErrorCode.OK']],
     ['batch_get_device_fp8', ['w8', 'x8s'], [131072, 3200], 'MxWide.BF16', ['ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device_fp8', ['h8'], [8192], 'MxWide.F16', ['ErrorCode.OK']],
     ['batch_get_device_fp8', ['f8', 'f8s'], [3072, 3072], 'MxWide.F32', ['ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device', ['w', 'pad8', 'x8s', 'f8s', 'kv'], [262144, 66, 3300, 3168, 16384],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', [262144, 66, 3300, 3168, 16384]]]],
    'get_into': [['batch_get',
      ['w#meta', 'kv#meta', 'w#meta', 'w8#meta', 'w8#meta', 'w8#meta', 'h8#meta', 'pad8#meta', 'x8s#meta', 'x8s#meta'],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK',
       'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_get_device', ['w'], [262144], ['ErrorCode.OK', [262144]]],
     ['batch_get_device_scatter', ['kv'], [2048], [4096], [8], ['ErrorCode.OK', [16384]]],
     ['batch_get_device_fp8_scatter', ['w8', 'w8', 'w8', 'x8s', 'x8s'], [131072, 131072, 131072, 3200, 3200],
      [131072, 512, 512, 64, 3200], [131072, 1024, 1024, 128, 3200], [1, 256, 256, 50, 1], 'MxWide.BF16',
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED', 'ErrorCode.NOT_IMPLEMENTED', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device_fp8', ['h8'], [8192], 'MxWide.F16', ['ErrorCode.OK']],
     ['batch_get', ['w#meta', 'pad8#meta', 'w8#meta', 'x8s#meta', 'x8s#meta'],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_get_device_fp8', ['w8', 'x8s', 'x8s'], [131072, 3200, 3200], 'MxWide.BF16',
      ['ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device', ['w', 'pad8', 'x8s', 'x8s'], [262144, 66, 3300, 3300],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', [262144, 66, 3300, 3300]]]],
    'rows': [['batch_get', ['w#meta', 'w8#meta', 'f8#meta', 'pad8#meta', 'x8s#meta', 'x8s#meta', 'f8s#meta', 'kv#meta', 'w#meta'],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK',
       'ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_get_device_fp8_range', ['w8', 'pad8', 'x8s', 'x8s'], [131072, 64, 3200, 3200], [5120, 18, 256, 0],
      [20480, 27, 320, 3200], 'MxWide.BF16',
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get', ['x8s#meta', 'x8s#meta'], ['ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_get_device_fp8', ['x8s', 'x8s'], [3200, 3200], 'MxWide.BF16',
      ['ErrorCode.NOT_IMPLEMENTED', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device', ['x8s', 'x8s'], [3300, 3300], ['ErrorCode.OK', 'ErrorCode.OK', [3300, 3300]]],
     ['batch_get_device_fp8_range', ['f8', 'f8s'], [3072, 3072], [288, 288], [2592, 2592], 'MxWide.F32',
      ['ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get', ['f8s#meta'], ['ErrorCode.OK']],
     ['batch_get_device_fp8', ['f8s'], [3072], 'MxWide.F32', ['ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device', ['f8s'], [3168], ['ErrorCode.OK', [3168]]],
     ['batch_get_device_range', ['w', 'kv', 'w'], [10240, 4096, 7168], [40960, 8192, 0],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['phases', [0, 0, 0, 4, 0, 0, 0, 0, 0]]],
    'slices': [['batch_get',
      ['kv#meta', 'kv#meta', 'kv#meta', 'kv#meta', 'kv8#meta', 'kv8#meta', 'kv8#meta', 'w8#meta', 'w#meta', 'pad8#meta',
       'h8#meta', 'f8#meta', 'x8s#meta', 'x8s#meta', 'f8s#meta', 'f8s#meta', 'kv8#meta'],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK',
       'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK',
       'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_get_device_fp8_range', ['f8s'], [3072], [96], [96], 'MxWide.F32', ['ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get', ['f8s#meta'], ['ErrorCode.OK']],
     ['batch_get_device_fp8', ['f8s'], [3072], 'MxWide.F32', ['ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device', ['f8s'], [3168], ['ErrorCode.OK', [3168]]],
     ['batch_get_device_fp8_range', ['kv8'], [8192], [4096], [4096], 'MxWide.BF16', ['ErrorCode.OK']],
     ['batch_get_device_range', ['kv'], [4096], [8192], ['ErrorCode.OK']],
     ['batch_get_device_fp8_strided', ['kv8', 'kv8', 'kv8', 'w8', 'pad8', 'x8s', 'x8s'],
      [8192, 8192, 8192, 131072, 64, 3200, 3200], [0, 512, 3, 3, 1, 8, 0], [1024, 512, 37, 57, 4, 16, 32],
      [2048, 1024, 64, 512, 9, 64, 64], [4, 8, 128, 256, 7, 50, 50], 'MxWide.BF16',
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED', 'ErrorCode.NOT_IMPLEMENTED', 'ErrorCode.NOT_IMPLEMENTED',
       'ErrorCode.NOT_IMPLEMENTED', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get', ['kv8#meta', 'w8#meta', 'pad8#meta', 'x8s#meta', 'x8s#meta'],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['batch_get_device_fp8', ['kv8', 'w8', 'x8s', 'x8s'], [8192, 131072, 3200, 3200], 'MxWide.BF16',
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device', ['pad8', 'x8s', 'x8s'], [66, 3300, 3300],
      ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', [66, 3300, 3300]]],
     ['batch_get_device_fp8_strided', ['h8'], [8192], [32], [64], [128], [64], 'MxWide.F16', ['ErrorCode.OK']],
     ['batch_get_device_fp8_strided', ['f8', 'f8s'], [3072, 3072], [4, 4], [16, 16], [96, 96], [32, 32], 'MxWide.F32',
      ['ErrorCode.OK', 'ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get', ['f8s#meta'], ['ErrorCode.OK']],
     ['batch_get_device_fp8', ['f8s'], [3072], 'MxWide.F32', ['ErrorCode.NOT_IMPLEMENTED']],
     ['batch_get_device', ['f8s'], [3168], ['ErrorCode.OK', [3168]]],
     ['batch_get_device_strided', ['kv', 'kv', 'kv', 'w'], [2048, 384, 10, 6], [2048, 1024, 64, 114], [4096, 2048, 128, 1024],
      [4, 8, 128, 256], ['ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK', 'ErrorCode.OK']],
     ['phases', [0, 0, 0, 10, 0, 0, 0, 0, 6, 0, 0, 0, 0, 0, 0, 0, 0]]],
}


@pytest.mark.parametrize("case", list(CASES))
def test_routes(env, case):
    cl, plain, store, rec, D, ref = env
    rec.log.clear()
    pairs = CASES[case](store, plain, D, ref)
    torch.cuda.synchronize()
    assert rec.log == EXPECTED[case]
    for j, (got, want) in enumerate(pairs):
        assert got.dtype == want.dtype and got.shape == want.shape, (case, j, got.shape, want.shape)
        assert torch.equal(_bits(got), _bits(want)), (case, j)
