"""Stream compaction: `nonzero`, `flatnonzero`, `argwhere`, `count_nonzero`, `extract` and `compress`, with NumPy 2.x's
results in C order on any number of ranks.

  * A rank's part of the condition (a box of the logical C-order array) is a set of equal-length RUNS of consecutive
    global positions (redistribute.block_runs).  rb200_compact_count counts the selected elements of every chunk of a
    run, rb200_cumulative scans the counts along each run (skipped when a run is one chunk), and rb200_compact writes
    every selected element's payload - a value, a flat index or its coordinates - from its run's base onwards.
  * The condition is read in place through this rank's strided view.  A pending input is instantiated first; an input
    whose parts overlap across ranks (a broadcast axis) is copied into a fresh array first, so no element is counted
    twice; `extract` also copies both operands when their parts differ on any rank.
  * One rank: count, scan, one synchronise to read the run totals, then compact straight into the result's shard.
  * Several ranks: one all-gather of the run totals (padded to the largest run count); every rank merges every rank's
    runs in global C order on the host (O(total runs)) and so knows every run's base; each rank compacts into a staging
    buffer in local order, which maps onto the output positions in increasing order.  One grouped send / receive moves
    each staging range to the rank that owns it in the result's default partition; pieces are placed with the op-list
    copy (`_pack_program`), consecutive pieces of one length at constant steps as one 2-D copy."""
import builtins
import operator

import numpy as np
import torch

from . import _cabi as cabi
from . import blocks
from . import common
from . import redistribute
from . import shardview
from .flush import _contig_strides, _pack_program
from .program import rb_dtype
from .runtime import RT, torch_dtype

_ZERO_D = "Calling nonzero on 0d arrays is not allowed. Use np.atleast_1d(scalar).nonzero() instead."


def _from_host(h):
    """A ramba array holding the host result h (the results of 0-d inputs), keeping h's dtype when h is empty."""
    from . import ramba as R

    return R.fromarray(h) if h.size else R.empty(h.shape, dtype=h.dtype)


def _cdiv(a, b):
    return -(-a // b)


def _fresh(a):
    """a copied into a new array of the engine's default partition."""
    from . import ramba as R

    new = R.empty(a.shape, dtype=a.dtype)
    R.DAG.assign(new, a)
    R.DAG.instantiate(new)
    return new


def _unmasked(a, what):
    if a.maskarray is not None:
        raise NotImplementedError("%s of a masked array" % what)


def _ready(*arrs, same_parts=False):
    """The inputs instantiated, and copied into fresh arrays when their parts overlap across ranks (or, with same_parts,
    when their parts are not the same boxes on every rank).  Every rank decides from the global distributions."""
    from . import ramba as R

    for a in arrs:
        R.DAG.instantiate(a)
    if common.num_workers == 1:
        return arrs
    copy = builtins.any(blocks.overlaps_across_ranks(a) for a in arrs)
    if same_parts and not copy:
        d0 = arrs[0].distribution
        for a in arrs[1:]:
            for s0, s1 in zip(d0, a.distribution):
                e0, e1 = shardview.is_empty(s0), shardview.is_empty(s1)
                if e0 != e1 or (not e0 and (list(s0.start) != list(s1.start) or list(s0.size) != list(s1.size))):
                    copy = True
    return tuple(_fresh(a) for a in arrs) if copy else arrs


def _runs(shape, sv):
    """(run starts in global C order, run length) of the part sv (None: the whole array) of an array of `shape`."""
    if sv is None:
        n = int(np.prod(shape))
        return np.zeros(1 if n else 0, dtype=np.int64), n
    if shardview.is_empty(sv):
        return np.zeros(0, dtype=np.int64), 0
    starts, length, _ = redistribute.block_runs(shape, [int(x) for x in sv.start], [int(x) for x in sv.size], True)
    return starts, length


def _device_i64(n):
    return torch.empty(max(n, 1), dtype=torch.int64, device=RT.device)


def _copy_pieces(code, isz, length, src_off, dst_off, sptr, dptr, dbounds):
    """Copy pieces (length, element offsets) from sptr to dptr: one 2-D strided op-list copy per run of equal lengths
    at constant steps."""
    prog = _pack_program(code, code)
    for (i0, cnt, ln, ds, dd) in redistribute.strided_groups(length, src_off, dst_off):
        RT.launch(prog, [cnt, ln], [0, 0], [(sptr + int(src_off[i0]) * isz, [ds, 1], code),
                                            (dptr + int(dst_off[i0]) * isz, [dd, 1], code, dbounds)])


def compact(cond, form, values=None):
    """The fresh 1-D result arrays of one compaction of `cond` (prepared by _ready): one int64 array of flat indices
    (cabi.COMPACT_FLAT), cond.ndim int64 coordinate arrays (COMPACT_COORDS), or one array of values' dtype holding the
    selected elements of `values` (COMPACT_VALUES, values prepared with cond)."""
    from . import ramba as R

    W, w = common.num_workers, common.worker_num
    shape = tuple(int(s) for s in cond.shape)
    dist = cond.distribution
    sv = None if W == 1 else dist[w]
    starts, run_len = _runs(shape, sv)
    n_runs = len(starts)
    cpr = _cdiv(run_len, cabi.COMPACT_CHUNK) if run_len else 0
    n_chunks = n_runs * cpr
    start = [0] * len(shape) if sv is None else [int(x) for x in sv.start]
    counts = _device_i64(n_chunks)
    cview = blocks.index_view(cond) if n_chunks else None
    ccode = rb_dtype(cond.dtype)
    keep = []
    if n_chunks:
        RT.compact_count(cview, ccode, run_len, counts.data_ptr())
    incl = counts
    if cpr > 1:
        incl = _device_i64(n_chunks)
        keep.append(RT.cumulative(counts.data_ptr(), incl.data_ptr(), cabi.I64, 1, cpr, n_runs, cabi.RED_ADD))
    totals = incl[(cpr - 1) * n_runs:cpr * n_runs] if n_chunks else incl[:0]
    if form == cabi.COMPACT_VALUES:
        dtypes = [values.dtype]
    else:
        dtypes = [np.dtype(np.int64)] * (len(shape) if form == cabi.COMPACT_COORDS else 1)
    if W == 1:
        tot = totals.cpu().numpy()
        bases = np.cumsum(tot) - tot
        N = int(tot.sum())
        outs = [R.empty((N,), dtype=dt) for dt in dtypes]
        ptrs = [blocks.block(o).ptr(0) for o in outs]
        if N:
            _launch_compact(cview, ccode, run_len, counts, incl, bases, form, values, start, shape, ptrs, keep)
        RT.hold(counts, incl, *keep)
        return outs
    # ---- several ranks: every rank's run totals, and the merge in global C order
    all_runs = [_runs(shape, s) for s in dist]
    maxr = builtins.max(builtins.max(len(s) for s, _ in all_runs), 1)
    mine = torch.zeros(maxr, dtype=torch.int64, device=RT.device)
    if n_runs:
        mine[:n_runs].copy_(totals)
    full = torch.empty(W * maxr, dtype=torch.int64, device=RT.device)
    RT.all_gather(full, mine).wait()
    allt = full.cpu().numpy().reshape(W, maxr)
    cat_starts = np.concatenate([s for s, _ in all_runs])
    cat_tot = np.concatenate([allt[r, :len(all_runs[r][0])] for r in range(W)])
    order = np.argsort(cat_starts, kind="stable")
    cat_base = np.empty_like(cat_tot)
    cat_base[order] = np.cumsum(cat_tot[order]) - cat_tot[order]
    first = np.cumsum([0] + [len(s) for s, _ in all_runs])
    base = [cat_base[first[r]:first[r + 1]] for r in range(W)]
    tots = [cat_tot[first[r]:first[r + 1]] for r in range(W)]
    N = int(cat_tot.sum())
    outs = [R.empty((N,), dtype=dt) for dt in dtypes]
    shards = [blocks.block(o) for o in outs]
    odist = outs[0].distribution

    def out_range(r):
        s = odist[r]
        if shardview.is_empty(s):
            return 0, 0
        return int(s.start[0]), int(s.size[0])

    my_tot = tots[w]
    my_loff = np.cumsum(my_tot) - my_tot
    n_mine = int(my_tot.sum())
    stage = [torch.empty(max(n_mine, 1), dtype=torch_dtype(dt), device=RT.device) for dt in dtypes]
    if n_mine:
        _launch_compact(cview, ccode, run_len, counts, incl, my_loff, form, values, start, shape, [s.data_ptr() for s in stage], keep)
    codes = [rb_dtype(dt) for dt in dtypes]
    isz = [blocks.itemsize(dt) for dt in dtypes]
    ops, unpack = [], []
    m0, mlen = out_range(w)
    for peer in range(W):
        p0, plen = out_range(peer)
        # my selected elements that `peer` owns: one contiguous range of my staging buffer
        ia, _, ps, pl = redistribute.intersect_runs(base[w], my_tot, np.array([p0], dtype=np.int64), plen)
        if len(ps):
            so = my_loff[ia] + (ps - base[w][ia])
            if peer == w:
                for st, sh, c, z in zip(stage, shards, codes, isz):
                    _copy_pieces(c, z, pl, so, ps - m0, st.data_ptr(), sh.ptr(0), sh.bounds)
            else:
                lo, hi = int(so[0]), int(so[-1] + pl[-1])
                ops += [(True, st[lo:hi], peer) for st in stage]
        if peer == w:
            continue
        # what I own of peer's selected elements
        ia, _, ps, pl = redistribute.intersect_runs(base[peer], tots[peer], np.array([m0], dtype=np.int64), mlen)
        if len(ps):
            n = int(pl.sum())
            bufs = [torch.empty(n, dtype=torch_dtype(dt), device=RT.device) for dt in dtypes]
            ops += [(False, b, peer) for b in bufs]
            unpack.append((pl, np.cumsum(pl) - pl, ps - m0, bufs))
    for wk in RT.p2p(ops):
        wk.wait()  # (the launching stream waits; the host does not)
    for (pl, so, do, bufs) in unpack:
        for b, sh, c, z in zip(bufs, shards, codes, isz):
            _copy_pieces(c, z, pl, so, do, b.data_ptr(), sh.ptr(0), sh.bounds)
    RT.hold(counts, incl, stage, ops, unpack, *keep)
    return outs


def _launch_compact(cview, ccode, run_len, counts, incl, bases, form, values, start, shape, ptrs, keep):
    run_base = torch.from_numpy(np.ascontiguousarray(bases, dtype=np.int64)).to(RT.device)
    keep.append(run_base)
    vview = blocks.index_view(values) if form == cabi.COMPACT_VALUES else None
    gstride = _contig_strides(shape)[0] if form == cabi.COMPACT_FLAT else None
    RT.compact(cview, ccode, run_len, counts.data_ptr(), incl.data_ptr(), run_base.data_ptr(), form, vview, start, gstride, ptrs)


# ---- the public functions ----------------------------------------------------------------------------------------------
def nonzero(a):
    """A tuple of a.ndim int64 arrays: the coordinates of a's nonzero elements in C order (NumPy's np.nonzero)."""
    from . import ramba as R

    a = R._as_nd(a)
    if not isinstance(a, R.ndarray):
        return np.nonzero(a)
    _unmasked(a, "nonzero")
    if a.ndim == 0:
        raise ValueError(_ZERO_D)
    (a,) = _ready(a)
    return tuple(compact(a, cabi.COMPACT_COORDS))


def flatnonzero(a):
    """The int64 flat C-order indices of a's nonzero elements (NumPy's np.flatnonzero)."""
    from . import ramba as R

    a = R._as_nd(a)
    if not isinstance(a, R.ndarray):
        return np.flatnonzero(a)
    _unmasked(a, "flatnonzero")
    if a.ndim == 0:
        return _from_host(np.flatnonzero(a.asarray()).astype(np.int64))
    (a,) = _ready(a)
    return compact(a, cabi.COMPACT_FLAT)[0]


def argwhere(a):
    """The (N, a.ndim) int64 array of the coordinates of a's nonzero elements (NumPy's np.argwhere)."""
    from . import ramba as R

    a = R._as_nd(a)
    if not isinstance(a, R.ndarray):
        return np.argwhere(a)
    _unmasked(a, "argwhere")
    if a.ndim == 0:
        return R.empty((1 if a.asarray() else 0, 0), dtype=np.int64)
    return R.stack(nonzero(a), axis=1)


def count_nonzero(a, axis=None, *, keepdims=False):
    """The number of nonzero elements of a, over every axis or along `axis` (NumPy's np.count_nonzero): the fused
    reduction of `a != 0` summed as int64."""
    from . import ramba as R

    a = R._as_nd(a)
    if not isinstance(a, R.ndarray):
        return np.count_nonzero(a, axis=axis, keepdims=keepdims)
    _unmasked(a, "count_nonzero")
    if a.ndim == 0:
        r = np.count_nonzero(a.asarray(), axis=axis, keepdims=keepdims)
        return R.array(r) if isinstance(r, np.ndarray) else r
    r = (a != 0).astype(np.int64).sum(axis=axis, keepdims=keepdims)
    if axis is None and not keepdims:
        return np.intp(r)
    return r


def extract(condition, arr):
    """The elements of arr where condition is nonzero, in C order (NumPy's np.extract), for operands of one shape."""
    from . import ramba as R

    arr = R._as_nd(arr)
    if not isinstance(arr, R.ndarray):
        if not isinstance(condition, R.ndarray):
            return np.extract(condition, arr)
        arr = R.fromarray(np.asarray(arr))
    if not isinstance(condition, R.ndarray):
        condition = R.fromarray(np.asarray(condition))
    if condition.shape != arr.shape:
        raise NotImplementedError("extract: condition of shape %s and array of shape %s (only operands of one shape are supported)"
                                  % (condition.shape, arr.shape))
    _unmasked(condition, "extract")
    _unmasked(arr, "extract")
    if arr.ndim == 0:
        return _from_host(np.extract(condition.asarray(), arr.asarray()))
    condition, arr = _ready(condition, arr, same_parts=True)
    return compact(condition, cabi.COMPACT_VALUES, arr)[0]


def compress(condition, a, axis=None):
    """The slices of a along `axis` (the flattened a for axis=None) where the 1-D condition is nonzero (NumPy's
    np.compress): a[..., flatnonzero(condition), ...] through integer-array indexing.  A condition shorter than the axis
    counts as False past its end; a nonzero entry past the end raises IndexError."""
    from . import ramba as R

    a = R._as_nd(a)
    if not isinstance(a, R.ndarray):
        a = R.fromarray(np.asarray(a))
    _unmasked(a, "compress")
    if isinstance(condition, R.ndarray):
        if condition.ndim != 1:
            raise ValueError("condition must be a 1-d array")
        idx = flatnonzero(condition)
    else:
        c = np.asarray(condition)
        if c.ndim != 1:
            raise ValueError("condition must be a 1-d array")
        idx = np.flatnonzero(c)
    if axis is None:
        a = R.reshape_copy(a, (a.size,))
        axis = 0
    else:
        if isinstance(axis, (bool, np.bool_)):
            raise TypeError("an integer is required for the axis")
        axis = operator.index(axis)
        if not -a.ndim <= axis < a.ndim:
            raise np.exceptions.AxisError(axis, a.ndim)
        axis %= a.ndim
    return a[(slice(None),) * axis + (idx,)]
