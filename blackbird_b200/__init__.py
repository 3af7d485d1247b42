"""blackbird_b200 — a Hopper-native tiered distributed object store.

Capabilities and API of blackbird-io/blackbird (Keystone control plane, striped + replicated
placement, TTL / soft-pin eviction, worker tiers, client SDK) with a data plane written for
one 8xH100 NVSwitch box: batched put/get run as hand-written sm_90a kernels that fuse the
NVLink transfer with a tensor-core checksum (TMA -> smem -> wgmma -> TMA).
"""
from . import _bb  # noqa: F401  (native core; must be built in-tree: python build.py)
from ._bb import ChecksumAlgo, ErrorCode  # noqa: F401

__version__ = "0.1.0"

_LAZY = {
    "LocalCluster": ("blackbird_b200.parallel", "LocalCluster"),
    "GpuRankCluster": ("blackbird_b200.parallel", "GpuRankCluster"),
    "CpuRankCluster": ("blackbird_b200.parallel", "CpuRankCluster"),
    "TensorStore": ("blackbird_b200.ops", "TensorStore"),            # imports torch
    "AsyncTensorStore": ("blackbird_b200.ops", "AsyncTensorStore"),
    "BlackbirdClient": ("blackbird_b200._bb", "BlackbirdClient"),
    "WorkerConfig": ("blackbird_b200._bb", "WorkerConfig"),
    "StorageClass": ("blackbird_b200._bb", "StorageClass"),
}


def __getattr__(name):  # lazy: `import blackbird_b200` must not import torch
    if name in _LAZY:
        import importlib

        mod, attr = _LAZY[name]
        return getattr(importlib.import_module(mod), attr)
    raise AttributeError(f"module 'blackbird_b200' has no attribute {name!r}")
