"""Binning: `histogram`, `histogram_bin_edges`, `bincount`, `searchsorted` and `digitize`, with NumPy 2.x's results on any
number of ranks.

  * The data are read in place through this rank's strided view (rb200_histogram, rb200_bin_search).  A pending input is
    instantiated first, an input whose parts overlap across ranks (a broadcast axis) is copied first, and data and
    weights whose parts differ on some rank are copied into one partition (compaction._ready); bool and integers
    narrower than 32 bits are widened by one fused copy, as for the index reductions.
  * Bin edges are NumPy's own: np.histogram_bin_edges runs on the host over a two-element stand-in holding the data's
    min and max (the engine's reductions) or over no data when the range is given, so NumPy raises its own
    errors.  Equal bins restate NumPy's fast path in the kernel, with the dtypes NumPy's promotion picks for each step.
  * histogram / bincount: every rank bins its own part into B partial counts (int64) or weight sums (float64); one
    sum all-reduce of B entries combines them at several ranks; each rank copies its block of the result out of it.
  * searchsorted / digitize: the sorted table goes to every device (a ramba table is gathered once); the result has
    v's shape and partition and is computed without an exchange."""
import builtins
import operator
import warnings

import numpy as np
import torch
from numpy.lib._histograms_impl import _get_outer_edges, _unsigned_subtract

from . import _cabi as cabi
from . import blocks
from . import common
from . import shardview
from .compaction import _ready, _unmasked
from .flush import _pack_program
from .program import rb_dtype
from .runtime import RT

_KERNEL_DTYPES = tuple(np.dtype(d) for d in (np.float64, np.float32, np.int64, np.int32))
_CMP = {np.dtype(np.float64): cabi.F64, np.dtype(np.float32): cabi.F32, np.dtype(np.int64): cabi.I64}


def _widen(a):
    """a, or one fused copy of it as int32 / int64 when its dtype is not one the kernels read."""
    if a.dtype in _KERNEL_DTYPES:
        return a
    return a.astype(np.int64 if a.dtype == np.uint32 else np.int32)


def _nd(x):
    from . import ramba as R

    x = R._as_nd(x)
    return x if isinstance(x, R.ndarray) else R.fromarray(np.asarray(x))


def _flat_nd(x):
    """x as a ramba array of at least one dimension (histogram flattens its input; a 0-d array keeps its value on the
    host)."""
    from . import ramba as R

    x = _nd(x)
    return R.fromarray(np.asarray(x.asarray()).reshape(1)) if x.ndim == 0 else x


def _host(x):
    from . import ramba as R

    return x.asarray() if isinstance(x, R.ndarray) else np.asarray(x)


def _min_max(a):
    """(min, max) of a as NumPy scalars of a's dtype: the engine's reductions (NaN when the data hold one)."""
    return a.dtype.type(a.min()), a.dtype.type(a.max())


# ---- bin edges ---------------------------------------------------------------------------------------------------------
def _stand_in(a, bins, range):
    """A host array that NumPy's edge computation treats as it treats a: a's dtype, and a's min and max when NumPy would
    look for them."""
    if np.ndim(bins) == 0 and range is None and a.size:
        return np.array(_min_max(a), dtype=a.dtype)
    return np.empty(0, dtype=a.dtype)


def _edges(a, bins, range):
    """(bin edges, (first, last, B) for equal bins or None), NumPy's own, with NumPy's errors."""
    if isinstance(bins, str):
        raise NotImplementedError("histogram: bins=%r needs percentiles; give a number of bins or the edges" % (bins,))
    if np.ndim(bins) != 0:
        bins = _host(bins)
    h = _stand_in(a, bins, range)
    edges = np.histogram_bin_edges(h, bins, range)
    if np.ndim(bins) != 0:
        return edges, None
    first, last = _get_outer_edges(h, range)
    return edges, (first, last, operator.index(bins))


def _bound(dtype, b):
    """(comparison dtype code, float value, int value) of NumPy's `x >= b` / `x <= b` for data of dtype."""
    if dtype.kind in "iub" and isinstance(b, (int, np.integer, np.bool_)):
        i = builtins.min(builtins.max(int(b), -(1 << 63)), (1 << 63) - 1)
        return cabi.I64, 0.0, i
    k = np.result_type(np.zeros(1, dtype), b)
    return _CMP[k], float(k.type(b)), 0


def _table_for(dtype, edges, uniform, dev_edges, cmp):
    """The cabi.BinTable of data of dtype binned by edges (on the device in cmp): equal bins restate NumPy's fast path
    with the dtypes its promotion picks for the subtraction, the division and the two range comparisons."""
    t = cabi.BinTable()
    t.n_bins = len(edges) - 1
    t.edges = dev_edges.data_ptr()
    t.edge_dtype = _CMP[np.dtype(cmp)]
    if uniform is None:
        t.form = cabi.BINS_EDGES
        return t
    first, last, n = uniform
    t.form = cabi.BINS_UNIFORM
    denom = _unsigned_subtract(last, first)
    s = _unsigned_subtract(np.zeros(1, edges.dtype), first)
    q = s / denom * n
    t.sub_dtype, t.div_dtype = _CMP[s.dtype], _CMP[q.dtype]
    t.first, t.denom = float(s.dtype.type(first)), float(q.dtype.type(denom))
    t.lo_dtype, t.lo, t.lo_i = _bound(dtype, first)
    t.hi_dtype, t.hi, t.hi_i = _bound(dtype, last)
    return t


def _edge_cmp(dtype, edges):
    """The dtype NumPy compares data of dtype with explicit edges in (searchsorted's common dtype)."""
    c = np.result_type(dtype, edges.dtype)
    if c.kind in "iub" and c != np.uint64:
        return np.dtype(np.int64)
    if c in (np.float64, np.float32):
        return c
    raise NotImplementedError("binning data of dtype %s against bins of dtype %s" % (dtype, edges.dtype))


def _sorted_table(table, cmp):
    """table converted to cmp on the device; NaN may only end it (NumPy's order)."""
    h = np.ascontiguousarray(table, dtype=cmp)
    if cmp.kind == "f":
        nan = np.isnan(h)
        if nan.any() and not nan[int(np.argmax(nan)):].all():
            raise NotImplementedError("bins or a sorted table with a NaN before a number")
    return torch.from_numpy(h.copy()).to(RT.device)


# ---- the kernels over every rank's part ----------------------------------------------------------------------------------
def _binned(src, w, table, B, out_dtype):
    """The ramba array of the B bins of src (weighted by w) over every rank, in out_dtype."""
    from . import ramba as R

    W = common.num_workers
    weighted = w is not None
    buf = torch.zeros(B, dtype=torch.float64 if weighted else torch.int64, device=RT.device)
    bad = torch.zeros(1, dtype=torch.int64, device=RT.device)
    keep = None
    sv = None if W == 1 else src.distribution[common.worker_num]
    if src.size and (sv is None or not shardview.is_empty(sv)):
        wview = blocks.index_view(w) if weighted else None
        keep = RT.histogram(blocks.index_view(src), rb_dtype(src.dtype), wview, rb_dtype(w.dtype) if weighted else 0, table,
                            buf.data_ptr(), bad.data_ptr())
    if W > 1:
        RT.all_reduce(buf, "sum")
    RT.hold(keep, table, bad)
    if int(bad.cpu()[0]):
        raise RuntimeError("histogram: %d elements fell outside every bin the host planned" % int(bad.cpu()[0]))
    res = R.empty((B,), dtype=out_dtype)
    rsv = res.distribution[common.worker_num]
    if not shardview.is_empty(rsv):
        sh = blocks.block(res)
        s0, n = int(rsv.start[0]), int(rsv.size[0])
        code = cabi.F64 if weighted else cabi.I64
        RT.launch(_pack_program(code, rb_dtype(out_dtype)), [n], [0], [(buf.data_ptr() + s0 * 8, [1], code), (sh.ptr(0), [1], rb_dtype(out_dtype), sh.bounds)])
    RT.hold(buf, keep)
    return res


def _weights_of(weights, what):
    w = _nd(weights)
    _unmasked(w, what)
    if w.dtype.kind not in "fiub":
        raise NotImplementedError("%s: weights of dtype %s" % (what, w.dtype))
    return w


# ---- the public functions ----------------------------------------------------------------------------------------------
def histogram_bin_edges(a, bins=10, range=None, weights=None):
    """NumPy's np.histogram_bin_edges of a (flattened), as a ramba array; string bins raise NotImplementedError."""
    from . import ramba as R

    a = _flat_nd(a)
    _unmasked(a, "histogram_bin_edges")
    if weights is not None and tuple(weights.shape if hasattr(weights, "shape") else np.shape(weights)) != tuple(a.shape):
        raise ValueError("weights should have the same shape as a.")
    edges, _ = _edges(_bool_as_uint8(a), bins, range)
    return R.fromarray(edges)


def _bool_as_uint8(a):
    if a.dtype == np.bool_:
        warnings.warn("Converting input from %s to %s for compatibility." % (a.dtype, np.dtype(np.uint8)), RuntimeWarning, stacklevel=4)
        return a.astype(np.uint8)
    return a


def histogram(a, bins=10, range=None, weights=None, density=False):
    """NumPy's np.histogram of a (flattened): (hist, bin_edges) as ramba arrays.  hist is int64 without weights and has
    the weights' dtype with them (summed in float64, then converted once)."""
    from . import ramba as R

    a = _flat_nd(a)
    _unmasked(a, "histogram")
    w = None
    if weights is not None:
        w = _weights_of(weights, "histogram")
        if w.ndim == 0 and a.shape == (1,):
            w = _flat_nd(w)
        if w.shape != a.shape:
            raise ValueError("weights should have the same shape as a.")
    a = _bool_as_uint8(a)
    edges, uniform = _edges(a, bins, range)
    B = len(edges) - 1
    cmp = edges.dtype if uniform is not None else _edge_cmp(a.dtype, edges)
    dev_edges = _sorted_table(edges, cmp)
    table = _table_for(a.dtype, edges, uniform, dev_edges, cmp)
    src = _widen(a)
    if w is not None:
        src, wk = _ready(src, _widen(w), same_parts=True)
    else:
        (src,) = _ready(src)
        wk = None
    hist = _binned(src, wk, table, B, np.dtype(np.int64) if w is None else w.dtype)
    RT.hold(dev_edges)
    if density:
        n = hist.asarray()
        db = np.array(np.diff(edges), float)
        hist = R.fromarray(n / db / n.sum())
    return hist, R.fromarray(edges)


def bincount(x, weights=None, minlength=0):
    """NumPy's np.bincount of the 1-D integer or bool x: int64 counts, or float64 sums of the weights converted to
    float64, of length max(max(x) + 1, minlength)."""
    from . import ramba as R

    x = R._as_nd(x)
    if not isinstance(x, R.ndarray) and not isinstance(weights, R.ndarray):
        return np.bincount(x, weights, minlength)
    x = _nd(x)
    _unmasked(x, "bincount")
    minlength = operator.index(minlength)
    if minlength < 0:
        raise ValueError("'minlength' must not be negative")
    if x.ndim != 1:
        raise ValueError("object too deep for desired array" if x.ndim > 1 else "object of too small depth for desired array")
    if not np.can_cast(x.dtype, np.intp, "safe"):
        raise TypeError("Cannot cast array data from %r to %r according to the rule 'safe'" % (x.dtype, np.dtype(np.intp)))
    w = None
    if weights is not None:
        w = _weights_of(weights, "bincount")
        if w.shape != x.shape:
            raise ValueError("The weights and list don't have the same length.")
    out_dtype = np.dtype(np.int64 if w is None else np.float64)
    if x.size == 0:
        return R.zeros((minlength,), dtype=out_dtype)
    lo, hi = _min_max(x)
    if lo < 0:
        raise ValueError("'list' argument must have no negative elements")
    B = builtins.max(int(hi) + 1, minlength)
    table = cabi.BinTable()
    table.form, table.n_bins = cabi.BINS_INTEGER, B
    src = _widen(x)
    if w is not None:
        src, wk = _ready(src, _widen(w), same_parts=True)
    else:
        (src,) = _ready(src)
        wk = None
    return _binned(src, wk, table, B, out_dtype)


def _side_code(side):
    if side not in ("left", "right"):
        raise ValueError("side must be 'left' or 'right' (got %r)" % (side,))
    return cabi.SEARCH_LEFT if side == "left" else cabi.SEARCH_RIGHT


def searchsorted(a, v, side="left", sorter=None):
    """NumPy's np.searchsorted of every element of v in the sorted 1-D a (a host array, or a ramba array gathered once):
    an int64 ramba array of v's shape and partition, np.intp for a scalar v.  Comparisons run in
    np.result_type(a, v), NaN after every number."""
    from . import ramba as R

    if sorter is not None:
        raise NotImplementedError("searchsorted: sorter= is not supported")
    a_h = _host(a)
    v = R._as_nd(v)
    if not isinstance(v, R.ndarray):
        return np.searchsorted(a_h, v, side=side)
    np.searchsorted(a_h, np.empty(0, dtype=v.dtype), side=side)  # NumPy's own checks of a and side
    code = _side_code(side)
    _unmasked(v, "searchsorted")
    if v.ndim == 0:
        return np.intp(np.searchsorted(a_h, v.asarray()[()], side=side))
    cmp = _edge_cmp(v.dtype, a_h)
    table = _sorted_table(a_h, cmp)
    (src,) = _ready(_widen(v))
    W = common.num_workers
    if W == 1:
        res = R.empty(v.shape, dtype=np.int64)
    else:
        dist = []
        for sv in src.distribution:
            if shardview.is_empty(sv):
                size, start = [0] * v.ndim, [0] * v.ndim
            else:
                size, start = [int(s) for s in sv.size], [int(s) for s in sv.start]
            dist.append(shardview.shardview(np.array(size, dtype=np.int64), np.array(start, dtype=np.int64)))
        res = R.create_array_with_divisions(v.shape, dist, dtype=np.int64)
    sv = None if W == 1 else src.distribution[common.worker_num]
    if src.size and (sv is None or not shardview.is_empty(sv)):
        sh = blocks.block(res)
        RT.bin_search(blocks.index_view(src), rb_dtype(src.dtype), table.data_ptr(), len(a_h), _CMP[cmp], code, sh.ptr(0))
    RT.hold(table)
    return res


def _monotonicity(bins):
    """NumPy's digitize rule on the bins as float64: 1 non-decreasing, -1 non-increasing (NumPy has checked the rest)."""
    d = np.asarray(bins, dtype=np.float64)
    diff = np.flatnonzero(d != d[0]) if d.size else np.zeros(0, dtype=np.int64)
    if not diff.size:
        return 1
    return 1 if d[0] < d[diff[0]] else -1


def digitize(x, bins, right=False):
    """NumPy's np.digitize: searchsorted of x in increasing bins, or in the reversed decreasing bins subtracted from
    len(bins)."""
    from . import ramba as R

    b = _host(bins)
    x = R._as_nd(x)
    if not isinstance(x, R.ndarray):
        return np.digitize(x, b, right=right)
    np.digitize(np.empty(0, dtype=x.dtype), b, right=right)  # NumPy's own checks of the bins
    side = "left" if right else "right"
    if _monotonicity(b) == -1:
        r = searchsorted(b[::-1], x, side=side)
        return len(b) - r
    return searchsorted(b, x, side=side)
