"""MXFP8 packing of fp16 and fp32 tensors on the GPU: the six client calls with `wide=` through GpuFabric, and
TensorStore round trips (contiguous, sliced and padded puts; get, get_into, get_rows, get_slice), every result equal to
the exact model of test_mxfp8_wide.py bit for bit, in the stored dtype."""
import numpy as np
import pytest
import torch

from test_mxfp8_exhaustive import model_unpack, same_bits
from test_mxfp8_wide import model_pack_w, model_unpack_w, same_wide

pytestmark = pytest.mark.gpu

NPU = {torch.float16: np.uint16, torch.float32: np.uint32}
W = {torch.float16: "f16", torch.float32: "f32"}


def _bits(t):
    torch.cuda.synchronize()
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu().numpy().view(NPU[t.dtype])


def _model(t):
    """The model's unpack(pack(t)) of a tensor's elements in row-major order (padded to whole blocks), as raw bits."""
    x = _bits(t).reshape(-1)
    n = x.size
    xp = np.concatenate([x, np.zeros(-n % 32, dtype=x.dtype)])
    return model_unpack_w(model_pack_w(xp, W[t.dtype]), xp.size, W[t.dtype])[:n].reshape(tuple(t.shape))


def _values(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = torch.randn(shape, generator=g, device="cuda") * torch.exp2(torch.randint(-10, 10, shape, generator=g, device="cuda").float())
    v.view(-1)[::101] = float("nan")
    v.view(-1)[3::257] = float("inf")
    return v.to(dtype)


@pytest.fixture(scope="module")
def cluster():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-fp8-wide")
    yield cl
    cl.stop()


def _cfg(bb, replicas=1):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=1, preferred_classes=[bb.StorageClass.RAM_GPU])


def test_six_client_calls(bb, cluster):
    """Put whole and gathered with 2 copies, then whole, range, strided and scattered gets, for fp16 and fp32."""
    c, s = cluster.client, torch.cuda.current_stream().cuda_stream
    OK = bb.ErrorCode.OK
    for dt in (torch.float16, torch.float32):
        wd = {torch.float16: bb.MxWide.F16, torch.float32: bb.MxWide.F32}[dt]
        per = 16 // torch.empty((), dtype=dt).element_size()
        rows, width = 2048, 24 * per
        n = rows * width
        x = _values((rows, width), dt, 1)
        big = torch.full((rows, width + 2 * per), float("nan"), dtype=dt, device="cuda")
        big[:, per:per + width] = x
        key = f"w/{W[dt]}"
        assert c.batch_put_device_fp8([key + "/a"], [x.data_ptr()], [n], _cfg(bb, 2), s, wide=wd) == [OK]
        v = big[:, per:per + width]
        assert c.batch_put_device_fp8_strided([key + "/g"], [v.data_ptr()], [width], [width + 2 * per], [rows], _cfg(bb), s, wide=wd) == [OK]
        want = _model(x)
        for k in (key + "/a", key + "/g"):
            out = torch.empty_like(x)
            assert c.batch_get_device_fp8([k], [out.data_ptr()], [n], s, wide=wd) == [OK]
            same_wide(_bits(out), want, W[dt], f"{k}: whole")
            lo, cnt = 3 * per, n // 3 + per
            buf = torch.full((cnt + 2 * per,), 7.0, dtype=dt, device="cuda")
            assert c.batch_get_device_fp8_range([k], [buf[per:].data_ptr()], [n], [lo], [cnt], s, wide=wd) == [OK]
            exp = np.concatenate([_bits(buf[:per]), want.reshape(-1)[lo:lo + cnt], _bits(buf[per + cnt:])])
            same_wide(_bits(buf), exp, W[dt], f"{k}: range")
            out = torch.empty((rows, 8 * per), dtype=dt, device="cuda")
            assert c.batch_get_device_fp8_strided([k], [out.data_ptr()], [n], [4 * per], [8 * per], [width], [rows], s, wide=wd) == [OK]
            same_wide(_bits(out), want[:, 4 * per:12 * per], W[dt], f"{k}: strided")
            dst = torch.full((rows, width + 2 * per), 7.0, dtype=dt, device="cuda")
            sv = dst[:, per:per + width]
            assert c.batch_get_device_fp8_scatter([k], [sv.data_ptr()], [n], [width], [width + 2 * per], [rows], s, wide=wd) == [OK]
            same_wide(_bits(sv), want, W[dt], f"{k}: scatter")
            assert (dst[:, :per] == 7).all() and (dst[:, per + width:] == 7).all(), f"{k}: scatter wrote a gap"


def test_tensor_store_round_trips(bb, cluster):
    """TensorStore with pack_fp8 for fp16 and fp32: contiguous, sliced (W[:, a:b], kv[:, :, h0:h1, :]) and padded puts;
    get, get_into (contiguous and a narrow), get_rows and get_slice along dims 0 and 1, in the stored dtype."""
    from blackbird_b200.ops.tensor_store import TensorStore

    store = TensorStore(cluster.client)
    for dt in (torch.float16, torch.float32):
        w = W[dt]
        Wt = _values((512, 96), dt, 2)
        kv = _values((4, 64, 8, 32), dt, 3)
        forms = {"c": Wt, "cols": Wt[:, 16:80], "heads": kv[:, :, 2:6, :], "pad": Wt[:333, :7]}
        for name, t in forms.items():
            key = f"ts/{w}/{name}"
            store.put(key, t, pack_fp8=True)
            want = _model(t)
            g = store.get(key)
            assert g.dtype == dt and tuple(g.shape) == tuple(t.shape), (key, g.dtype)
            same_wide(_bits(g), want, w, f"{key}: get")
            out = torch.empty_like(t.contiguous())
            store.get_into(key, out)
            same_wide(_bits(out), want, w, f"{key}: get_into")
            host = torch.full((t.shape[0], t.shape[1] + 16) + tuple(t.shape[2:]), 5.0, dtype=dt, device="cuda")
            nar = host.narrow(1, 8, t.shape[1])
            store.get_into(key, nar)
            same_wide(_bits(nar), want, w, f"{key}: get_into narrow")
            assert (host[:, :8] == 5).all() and (host[:, 8 + t.shape[1]:] == 5).all(), key
            a, b = t.shape[0] // 3, min(t.shape[0], t.shape[0] // 3 + 37)
            r = store.get_rows(key, a, b)
            assert r.dtype == dt
            same_wide(_bits(r), want[a:b], w, f"{key}: get_rows")
            for d, (s0, s1) in ((0, (t.shape[0] // 4, t.shape[0] - t.shape[0] // 5)), (1, (1, t.shape[1] - 2))):
                sl = store.get_slice(key, d, s0, s1)
                same_wide(_bits(sl), np.take(want, range(s0, s1), axis=d), w, f"{key}: get_slice dim {d}")
        store.remove([f"ts/{w}/{n}" for n in forms])


def test_fp32_object_read_as_bf16_and_type_errors(bb, cluster):
    """An fp32-packed object read with wide=BF16 is the model's bf16 unpack; pack_fp8 on int / fp64 is a TypeError."""
    from blackbird_b200.ops.tensor_store import TensorStore

    c, s = cluster.client, torch.cuda.current_stream().cuda_stream
    x = _values((64, 256), torch.float32, 4)
    n = x.numel()
    assert c.batch_put_device_fp8(["x32"], [x.data_ptr()], [n], _cfg(bb), s, wide=bb.MxWide.F32) == [bb.ErrorCode.OK]
    out = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    assert c.batch_get_device_fp8(["x32"], [out.data_ptr()], [n], s) == [bb.ErrorCode.OK]
    torch.cuda.synchronize()
    packed = model_pack_w(_bits(x).reshape(-1), "f32")
    same_bits(out.view(torch.int16).cpu().numpy(), model_unpack(packed, n), "bf16", "fp32 object read as bf16")
    store = TensorStore(c)
    for bad in (torch.zeros(64, dtype=torch.int32, device="cuda"), torch.zeros(64, dtype=torch.float64, device="cuda")):
        with pytest.raises(TypeError):
            store.put("bad", bad, pack_fp8=True)


def test_mixed_dtype_batch_through_tensor_store(bb, cluster):
    """A batch of bf16, fp16 and fp32 tensors makes one fused call per dtype and returns each in its dtype."""
    from blackbird_b200.ops.tensor_store import TensorStore

    store = TensorStore(cluster.client)
    ts = [_values((128, 64), dt, 5 + i) for i, dt in enumerate((torch.bfloat16, torch.float16, torch.float32))]
    keys = [f"mix/{i}" for i in range(3)]
    store.batch_put(keys, ts, pack_fp8=True)
    got = store.batch_get(keys)
    assert [g.dtype for g in got] == [t.dtype for t in ts]
    for t, g in zip(ts[1:], got[1:]):
        same_wide(_bits(g), _model(t), W[t.dtype], f"mixed batch {t.dtype}")
    torch.cuda.synchronize()
    from test_mxfp8_exhaustive import model_pack

    xb = ts[0].view(torch.int16).cpu().numpy().view(np.uint16).reshape(-1)
    same_bits(got[0].view(torch.int16).cpu().numpy(), model_unpack(model_pack(xb), xb.size).reshape(128, 64), "bf16", "mixed bf16")
