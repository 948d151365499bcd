"""ramba_b200.blocks — this rank's block of an array, for the operations that write or read it outside a fused op (the
uploads, the constant fill, the host copies, stage 2 of reductions, reshape_copy, the scan, integer-array indexing,
groupby).

They share one rule: a block written or read outside a flush is created at the array's current partition, and that
partition is then fixed.  A flush pins a flexible partition to its op's and reuses a block that already exists, so a
block made at the old partition and left flexible would be addressed with the wrong box.  Like flush.py, this module
depends on the runtime and the partition algebra only, never on the array API in ramba.py.
"""
import builtins

import numpy as np

from . import _cabi as cabi
from . import common
from . import shardview
from .flush import _local_shape
from .runtime import RT


def block(nd):
    """This rank's Shard of nd's storage (created at the array's current partition on first use); fixes the partition."""
    bd = nd.bdarray
    sh = RT.shards.get(nd.gid) or RT.create_array(nd.gid, _local_shape(bd.distribution, common.worker_num), bd.dtype, bd.pad)
    bd.remote_constructed = True
    bd.flex_dist = False
    return sh


def part(nd):
    """This rank's part of view nd: (device address, element strides, allocation bounds, shape)."""
    sv = nd.distribution[common.worker_num]
    sh = block(nd)
    off, st = RT.bind_view(sv, sh.strides, shardview.clean_range(sv))
    return sh.ptr(off), st, sh.bounds, [int(x) for x in sv.size]


def itemsize(dtype):
    """Bytes of one stored element (bool is stored as uint8)."""
    return np.dtype(np.uint8 if dtype == np.bool_ else dtype).itemsize


def index_view(nd):
    """IndexView of this rank's part of view nd (the whole view at one rank)."""
    ptr, st, bounds, shape = part(nd)
    return cabi.index_view(ptr, shape, st, itemsize(nd.dtype), bounds)


def flat_index_view(nd):
    """1-D IndexView over this rank's whole shard of nd, indexed by element offsets from its interior origin."""
    sh = block(nd)
    n = sh.buf.numel() - sh.origin
    return cabi.index_view(sh.ptr(0), [n], [1], itemsize(nd.dtype), sh.bounds)


def overlaps_across_ranks(nd):
    """True when the parts of view nd on different ranks share elements (a broadcast axis of length > 1)."""
    return builtins.any(int(sv.axis_map[d]) < 0 and nd.shape[d] > 1 for sv in nd.distribution if not shardview.is_empty(sv)
                        for d in range(len(nd.shape)))
