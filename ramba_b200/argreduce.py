"""First-occurrence index reductions: `argmax`, `argmin`, `nanargmax` and `nanargmin`, globally and along one axis, with
NumPy 2.x's results on any number of ranks.

  * The source is read in place through this rank's strided view (slices, steps, reversals, transposes, broadcast axes,
    padded shards).  A pending expression is instantiated first; bool and integers narrower than 32 bits are widened by
    one fused copy (uint32 to int64), so that the kernel reads float64, float32, int64 or int32 only.
  * rb200_arg_reduce gives every output its global index and its order key (include/ramba_b200.h): the view's origin in
    the global array and the global C-order strides go with the call, so nothing is renumbered afterwards.
  * One rank: no collective; a result over every axis is one 8-byte read to the host.
  * Several ranks, two layouts.  When the axis is not cut across ranks (and no rank's part overlaps another's), each
    rank's output is its block of the result, partitioned like the source over the kept axes: nothing is exchanged.
    Otherwise (also for every axis at once) each rank packs its (key, index) pairs into buffers of the result's global
    shape holding (INT64_MIN, INT64_MAX) elsewhere; one max all-reduce of the keys, the indices whose key is not the
    global one set to INT64_MAX, one min all-reduce of the indices: two collectives of 8 bytes per result element.
    The same logical element has the same key and index on every rank, so overlapping broadcast views need no copy.
  * A nan variant whose slice holds only NaN leaves INT64_MAX, which raises ValueError.  In the layout without an
    exchange that check takes one 8-byte max all-reduce so that every rank raises together."""
import builtins
import operator

import numpy as np
import torch

from . import _cabi as cabi
from . import blocks
from . import common
from . import shardview
from .flush import _contig_strides, _pack_program
from .program import E, Lowering, rb_dtype
from .runtime import RT

NO_INDEX = int(np.iinfo(np.int64).max)
KEY_MIN = int(np.iinfo(np.int64).min)
_KERNEL_DTYPES = tuple(np.dtype(d) for d in (np.float64, np.float32, np.int64, np.int32))
_OPS = {"argmax": cabi.ARG_MAX, "argmin": cabi.ARG_MIN, "nanargmax": cabi.ARG_NANMAX, "nanargmin": cabi.ARG_NANMIN}

_mask_prog = []


def _mask_program():
    """idx = key == global_key ? idx : INT64_MAX; views: idx, key, global_key (int64)."""
    if not _mask_prog:
        lw = Lowering([cabi.I64, cabi.I64, cabi.I64])
        v = lw.build(E("where", E("eq", lw.read_view(1), lw.read_view(2)), lw.read_view(0), lw.scalar(NO_INDEX)), None)
        lw.store(0, v)
        _mask_prog.append(lw.finish())
    return _mask_prog[0]


def _device_i64(n, fill=None):
    if fill is None:
        return torch.empty(max(n, 1), dtype=torch.int64, device=RT.device)
    return torch.full((max(n, 1),), fill, dtype=torch.int64, device=RT.device)


def _source(a):
    from . import ramba as R

    if a.dtype not in _KERNEL_DTYPES:  # bool and narrow integers: one fused widening copy
        a = a.astype(np.int64 if a.dtype == np.uint32 else np.int32)
    R.DAG.instantiate(a)
    return a


def _block(src):
    """(holds a part, start, size) of this rank's part of the source (at one rank: the whole source)."""
    if common.num_workers == 1:
        return True, [0] * src.ndim, [int(x) for x in src.shape]
    sv = src.distribution[common.worker_num]
    return not shardview.is_empty(sv), [int(x) for x in sv.start], [int(x) for x in sv.size]


def _kernel(src, axis, op, start, out_idx, out_key):
    """rb200_arg_reduce of this rank's part of src; returns what the launch keeps alive."""
    return RT.arg_reduce(blocks.index_view(src), rb_dtype(src.dtype), axis, op, start, _contig_strides(src.shape)[0], out_idx, out_key)


def _max_index(ptr, n):
    """A 1-element device tensor holding the largest of the n int64 at ptr (INT64_MIN when n == 0): the order key of
    rb200_arg_reduce's ARG_MAX over them."""
    idx, key = _device_i64(1), _device_i64(1, KEY_MIN)
    keep = None
    if n:
        keep = RT.arg_reduce(cabi.index_view(ptr, [n], [1], 8), cabi.I64, cabi.ARG_ALL_AXES, cabi.ARG_MAX, [0], [1], idx.data_ptr(), key.data_ptr())
    RT.hold(idx, keep)
    return key


def _exchange(lidx, lkey, lshape, lstart, rshape, n_loc):
    """The global result (flat int64 tensor of shape rshape) from every rank's (index, key) block at lstart."""
    n = int(np.prod(rshape))
    gidx, gkey = _device_i64(n, NO_INDEX), _device_i64(n, KEY_MIN)
    gst = _contig_strides(rshape)[0]
    lst = _contig_strides(lshape)[0]
    off = builtins.sum(s * st for s, st in zip(lstart, gst)) * 8
    z = [0] * len(lshape)
    if n_loc:
        RT.launch(_pack_program(cabi.I64, cabi.I64), lshape, z, [(lkey.data_ptr(), lst, cabi.I64), (gkey.data_ptr() + off, gst, cabi.I64)])
    RT.all_reduce(gkey, "max")
    if n_loc:
        RT.launch(_mask_program(), lshape, z,
                  [(lidx.data_ptr(), lst, cabi.I64), (lkey.data_ptr(), lst, cabi.I64), (gkey.data_ptr() + off, gst, cabi.I64)])
        RT.launch(_pack_program(cabi.I64, cabi.I64), lshape, z, [(lidx.data_ptr(), lst, cabi.I64), (gidx.data_ptr() + off, gst, cabi.I64)])
    RT.all_reduce(gidx, "min")
    RT.hold(lidx, lkey, gkey)
    return gidx


def _all_nan():
    raise ValueError("All-NaN slice encountered")


def _global(a, op, checks_nan):
    """The flat index over every axis of a non-empty array, as a Python int."""
    src = _source(a)
    holds, start, _ = _block(src)
    idx, key = _device_i64(1), _device_i64(1)
    keep = _kernel(src, cabi.ARG_ALL_AXES, op, start, idx.data_ptr(), key.data_ptr()) if holds else None
    if common.num_workers > 1:
        idx = _exchange(idx, key, [1], [0], [1], 1 if holds else 0)
    RT.hold(keep)
    i = int(idx.cpu()[0])
    if checks_nan and i == NO_INDEX:
        _all_nan()
    return i


def _axis_cut(src, ax):
    L = src.shape[ax]
    return builtins.any(not shardview.is_empty(sv) and (int(sv.start[ax]) != 0 or int(sv.size[ax]) != L) for sv in src.distribution)


def _along(a, axis, op, checks_nan, keepdims):
    """The int64 ramba array of positions along `axis` (a.shape[axis] > 0, a non-empty result)."""
    from . import ramba as R

    src = _source(a)
    W = common.num_workers
    cut = W > 1 and (_axis_cut(src, axis) or blocks.overlaps_across_ranks(src))
    rshape = tuple(s for d, s in enumerate(src.shape) if d != axis)
    fshape = tuple(1 if d == axis else s for d, s in enumerate(src.shape)) if keepdims else rshape
    holds, bstart, bsize = _block(src)
    lshape = [s for d, s in enumerate(bsize) if d != axis]
    lstart = [s for d, s in enumerate(bstart) if d != axis]
    n_loc = int(np.prod(lshape)) if holds else 0
    if not cut:
        if W == 1:
            res = R.empty(fshape, dtype=np.int64)
        else:
            dist = []
            for sv in src.distribution:
                if shardview.is_empty(sv):
                    size, start = [0] * len(fshape), [0] * len(fshape)
                else:
                    size = [1 if d == axis else int(x) for d, x in enumerate(sv.size) if keepdims or d != axis]
                    start = [0 if d == axis else int(x) for d, x in enumerate(sv.start) if keepdims or d != axis]
                dist.append(shardview.shardview(np.array(size, dtype=np.int64), np.array(start, dtype=np.int64)))
            res = R.create_array_with_divisions(fshape, dist, dtype=np.int64)
        sh = blocks.block(res)
        key = _device_i64(n_loc)
        keep = _kernel(src, axis, op, bstart, sh.ptr(0), key.data_ptr()) if n_loc else None
        RT.hold(key, keep)
        if checks_nan:
            worst = _max_index(sh.ptr(0), n_loc)
            if W > 1:
                RT.all_reduce(worst, "max")
            if int(worst.cpu()[0]) == NO_INDEX:
                _all_nan()
        return res
    lidx, lkey = _device_i64(n_loc), _device_i64(n_loc)
    keep = _kernel(src, axis, op, bstart, lidx.data_ptr(), lkey.data_ptr()) if n_loc else None
    gidx = _exchange(lidx, lkey, lshape, lstart, rshape, n_loc)
    if checks_nan and int(_max_index(gidx.data_ptr(), int(np.prod(rshape))).cpu()[0]) == NO_INDEX:
        _all_nan()
    res = R.empty(fshape, dtype=np.int64)
    sv = res.distribution[common.worker_num]
    if not shardview.is_empty(sv):
        sh = blocks.block(res)
        size = [int(x) for x in sv.size]
        start = [int(x) for x in sv.start]
        gst = _contig_strides(rshape)[0]
        if keepdims:
            gst = gst[:axis] + [0] + gst[axis:]
        off = builtins.sum((0 if keepdims and d == axis else s) * gst[d] for d, s in enumerate(start)) * 8
        RT.launch(_pack_program(cabi.I64, cabi.I64), size, [0] * len(size),
                  [(gidx.data_ptr() + off, gst, cabi.I64), (sh.ptr(0), _contig_strides(size)[0], cabi.I64, sh.bounds)])
    RT.hold(gidx, keep)
    return res


def arg_reduce(a, name, axis=None, out=None, keepdims=False):
    """argmax / argmin / nanargmax / nanargmin of `a` with NumPy's signature and results: an int64 NumPy scalar for
    axis=None (the flat C-order index in the logical shape), an int64 ramba array for an axis."""
    from . import ramba as R

    a = R._as_nd(a)
    if not isinstance(a, R.ndarray):  # Python scalars and sequences
        return getattr(np, name)(a, axis=axis, out=out, keepdims=keepdims)
    if out is not None:
        raise NotImplementedError("%s: out= is not supported" % name)
    if a.maskarray is not None:
        raise NotImplementedError("%s of a masked array" % name)
    op = _OPS[name]
    base = name[3:] if name.startswith("nan") else name
    checks_nan = op in (cabi.ARG_NANMAX, cabi.ARG_NANMIN) and a.dtype.kind == "f"
    if axis is not None:
        if isinstance(axis, (bool, np.bool_)):
            raise TypeError("an integer is required for the axis")
        axis = operator.index(axis)  # a tuple or a float raises TypeError, as in NumPy
        nd = builtins.max(a.ndim, 1)
        if not -nd <= axis < nd:
            raise np.exceptions.AxisError(axis, nd)
        axis %= nd
    if a.ndim == 0:
        if checks_nan and np.isnan(a.asarray()):
            _all_nan()
        return np.int64(0)
    if axis is None or a.ndim == 1:
        if a.size == 0:
            raise ValueError("attempt to get %s of an empty sequence" % base)
        i = _global(a, op, checks_nan)
        return R.full((1,) * a.ndim, i, dtype=np.int64) if keepdims else np.int64(i)
    if a.shape[axis] == 0:
        raise ValueError("attempt to get %s of an empty sequence" % base)
    if builtins.any(s == 0 for d, s in enumerate(a.shape) if d != axis):
        return R.empty(tuple(1 if d == axis else s for d, s in enumerate(a.shape)) if keepdims else
                       tuple(s for d, s in enumerate(a.shape) if d != axis), dtype=np.int64)
    return _along(a, axis, op, checks_nan, keepdims)
