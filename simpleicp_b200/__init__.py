"""simpleicp_b200 — H100-native (sm_90a) point-to-plane ICP with the simpleICP Python API.

Drop-in names of the reference package (python/simpleicp/__init__.py:12-14):
``SimpleICP``, ``PointCloud``, ``RigidBodyParameters``; plus the functional form
``simpleicp(X_fix, X_mov, **kwargs)`` and the batched / multi-GPU ``simpleicp_batch``.
"""
__version__ = "0.1.0"

import logging as _logging

_logging.getLogger(__name__).addHandler(_logging.NullHandler())

from .simpleicp import SimpleICP, SimpleICPException, simpleicp, register  # noqa: E402
from .pointcloud import PointCloud, PointCloudException  # noqa: E402
from .optimization import RigidBodyParameters, Parameter  # noqa: E402
from .batch import simpleicp_batch, shard_pairs, tile_slabs, close_engine_pool  # noqa: E402
from ._capi import read_xyz, write_xyz  # noqa: E402
from .linearized import simpleicp_linearized  # noqa: E402

__all__ = [
    "SimpleICP", "SimpleICPException", "PointCloud", "PointCloudException", "RigidBodyParameters",
    "Parameter", "simpleicp", "simpleicp_linearized", "register", "simpleicp_batch", "shard_pairs", "tile_slabs", "close_engine_pool", "read_xyz", "write_xyz",
]
