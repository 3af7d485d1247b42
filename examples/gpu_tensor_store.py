#!/usr/bin/env python3
"""GPU tier from torch (needs H100s): one process per GPU, `torchrun --nproc-per-node N examples/gpu_tensor_store.py`.
Every rank puts activations on its ring neighbour, reads its neighbour's back, stores a KV block as MXFP8 (pack fused
into the put kernel) and reads it back (unpack fused into the get kernel)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from blackbird_b200 import _bb  # noqa: E402
from blackbird_b200.ops import TensorStore  # noqa: E402
from blackbird_b200.parallel import GpuRankCluster  # noqa: E402


def main():
    cl = GpuRankCluster(slab_bytes=2 << 30)
    nxt = (cl.rank + 1) % cl.world
    store = TensorStore(cl.client, _bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, preferred_node=f"gpu{nxt}",
                                                    preferred_classes=[_bb.StorageClass.RAM_GPU], ttl_ms=0))
    act = torch.randn(4096, 4096, device="cuda")
    store.put(f"act/{cl.rank}", act)                       # one fused launch: NVLink copy + tensor-core digest
    cl.barrier()
    prev = (cl.rank - 1) % cl.world
    got = store.get(f"act/{prev}")                         # verified against the digest recorded at put time
    kv = (torch.randn(64, 16384, device="cuda") * 2).to(torch.bfloat16)
    store.put(f"kv/{cl.rank}", kv, pack_fp8=True)          # bf16 read once, 0.52x the bytes cross NVLink
    back = store.get(f"kv/{cl.rank}")
    err = (back.float() - kv.float()).abs().max().item() / kv.float().abs().max().item()
    print(f"rank {cl.rank}: read act/{prev} {tuple(got.shape)}, MXFP8 round trip max rel err {err:.4f}, launches {cl.fabric.launches}")
    cl.barrier()
    store.remove([f"act/{cl.rank}", f"kv/{cl.rank}"])
    cl.stop()


if __name__ == "__main__":
    main()
