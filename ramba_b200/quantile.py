"""Order statistics: `median`, `percentile`, `quantile` and their nan variants, with NumPy 2.x's signatures and results on
any number of ranks.

  * The device finds which keys sit at which ranks (rb200_select_*: a radix select over the order-preserving key map of
    include/ramba_b200.h); every value is then finished on the host with NumPy's own arithmetic over the selected values
    only (at most 2 * len(q) per output): np.mean of the one or two middle values for a median, NumPy's
    _QuantileMethods / _get_indexes / _get_gamma / _lerp for a quantile, with the slice length as a Python int as NumPy
    has it.  nanmedian along an axis shorter than 600 of an array of two or more dims is finished as NumPy's masked-array
    path does it (an odd count adds the middle value to itself and halves the sum, so two float32 values near FLT_MAX
    give inf there).  So every result equals NumPy's with ==.  The one exception is the sign of a zero when -0.0 and +0.0 tie at a selected rank: the key order puts -0.0 first,
    while NumPy's partition treats the two as equal, so either zero may come back.
  * The source is read in place through this rank's strided view; a pending input is instantiated first, an input whose
    parts overlap across ranks is copied first, and bool and integers narrower than 32 bits are widened by one fused copy
    (uint32 to int64), as for the index reductions.  The reduced axis becomes the view's last dim, so each output
    position is one segment.
  * Forms (the library picks one from the shapes): `row` when a segment fits in shared memory (one launch, one read of
    the data; the ranks of a nan variant come from a table indexed by the segment's count of numbers), `pass` otherwise:
    one count pass and one choose per digit, the nan counts read once after pass 0 to place the ranks, and for a single
    segment a switch to candidate compaction once few enough keys still match.
  * Several ranks: an axis that is not cut (and parts that do not overlap) is computed by each rank for its own segments,
    the result partitioned like the source over the kept axes, with no exchange.  Otherwise (every axis at once, or a
    cut axis) each rank counts its part of every segment into count rows of the global segments and one sum all-reduce
    of the counts follows each pass (and of the nan counts after pass 0), so every rank chooses the same buckets and
    ends with the same keys without moving any data."""
import builtins
import operator
import warnings

import numpy as np
import torch
from numpy.lib import _function_base_impl as fnb

from . import _cabi as cabi
from . import blocks
from . import common
from . import shardview
from .argreduce import _KERNEL_DTYPES, _device_i64, _source
from .compaction import _ready, _unmasked
from .flush import _contig_strides, _pack_program
from .program import rb_dtype
from .runtime import RT

_HOST_DTYPES = _KERNEL_DTYPES + tuple(np.dtype(d) for d in (np.int16, np.int8, np.uint32, np.uint16, np.uint8, np.bool_))


# ---- the key map (include/ramba_b200.h), host side --------------------------------------------------------------------
def keys_of(x):
    """The order-preserving uint64 key of every element of a float64 / float32 / int64 / int32 array."""
    x = np.asarray(x)
    if x.dtype == np.float64 or x.dtype == np.float32:
        bits = 64 if x.dtype == np.float64 else 32
        u = x.view(np.uint64 if bits == 64 else np.uint32).astype(np.uint64)
        sign = np.uint64(1 << (bits - 1))
        full = np.uint64((1 << bits) - 1)
        k = np.where(u & sign, ~u & full, u | sign)
        return np.where(np.isnan(x), full, k).astype(np.uint64)
    if x.dtype == np.int64:
        return x.view(np.uint64) ^ np.uint64(1 << 63)
    return (x.view(np.uint32) ^ np.uint32(1 << 31)).astype(np.uint64)


def values_of(keys, dtype):
    """The inverse of keys_of: the values of dtype whose keys these are (a NaN key gives the default quiet NaN)."""
    k = np.asarray(keys, dtype=np.uint64)
    dtype = np.dtype(dtype)
    if dtype.kind == "f":
        bits = 64 if dtype == np.float64 else 32
        sign = np.uint64(1 << (bits - 1))
        full = np.uint64((1 << bits) - 1)
        u = np.where(k & sign, k ^ sign, ~k & full)
        v = u.astype(np.uint64 if bits == 64 else np.uint32).view(dtype)
        return np.where(k == full, dtype.type(np.nan), v)
    if dtype == np.int64:
        return (k ^ np.uint64(1 << 63)).view(np.int64)
    return (k.astype(np.uint32) ^ np.uint32(1 << 31)).view(np.int32)


# ---- which ranks a result needs (NumPy's own index rules) -----------------------------------------------------------------
class _Spec:
    """What one call asks for: median (kind "median") or quantiles q (a NumPy array, NumPy's dtype) by method; masked:
    a median finished as numpy.ma.median finishes it (NumPy's nanmedian along a short axis)."""

    def __init__(self, kind, q=None, method="linear", masked=False):
        self.kind, self.q, self.method, self.masked = kind, q, method, masked
        self.qf = None if q is None else q.reshape(-1)
        self.props = None if q is None else fnb._QuantileMethods[method]

    @property
    def K(self):
        if self.kind == "median":
            return 2
        return self.qf.size * (1 if self._integral() else 2)

    def _integral(self):
        if self.props["fix_gamma"] is None:
            return True
        vi = np.asanyarray(self.props["get_virtual_index"](2, self.qf))
        return self.method == "linear" and np.issubdtype(vi.dtype, np.integer)

    def _exact_below(self):
        """Counts below this are exact in q's dtype, so that a count array converted to it gives the virtual indexes a
        Python int gives (NumPy converts the Python int n, or n - 1, to q's dtype once)."""
        if self.qf.dtype.kind != "f":
            return 1 << 62
        return 1 << (np.finfo(self.qf.dtype).nmant + 1)

    def indexes(self, n, data_dtype):
        """(indexes into the sorted slice of n numbers, shape (..., K), or -1 for the last; virtual indexes) for n a
        Python int (NumPy's arithmetic exactly) or an int64 array of counts below _exact_below()."""
        if self.kind == "median":
            n = np.asarray(n, dtype=np.int64)
            return np.stack([(n - 1) // 2, n // 2], axis=-1), None
        if not isinstance(n, int):
            n = np.asarray(n)
            assert n.size == 0 or int(n.max()) < self._exact_below()
            n = n[..., None]
            if self.qf.dtype.kind == "f":
                n = n.astype(self.qf.dtype)
        vi = np.asanyarray(self.props["get_virtual_index"](n, self.qf))
        if self._integral():
            return vi.astype(np.intp), vi
        prev, nxt = fnb._get_indexes(np.empty(0, data_dtype), vi, n)
        return np.concatenate([prev, nxt], axis=-1), vi

    def ranks(self, nv, data_dtype):
        """The ranks (int64, shape nv.shape + (K,)) to select for slices of nv numbers (0 where nv == 0): NumPy's indexes
        for each distinct count, computed over an array of the counts while they are exact in q's dtype and with each
        count as a Python int beyond."""
        nv = np.asarray(nv, dtype=np.int64)
        u, inv = np.unique(nv, return_inverse=True)
        if self.kind == "median" or u[-1] < self._exact_below():
            idx = np.broadcast_to(self.indexes(u, data_dtype)[0], u.shape + (self.K,))
        else:
            idx = np.stack([self.indexes(int(n), data_dtype)[0] for n in u])
        idx = idx.astype(np.int64)
        last = np.maximum(u - 1, 0)[..., None]
        return np.clip(np.where(idx < 0, last, idx), 0, last)[inv.reshape(nv.shape)]

    def finish(self, vals, n, data_dtype, used):
        """The results (G, len(q)) or (G,) of G slices of n numbers whose selected values are vals (G, K), with NumPy's
        arithmetic; used: the ranks the device selected, checked against NumPy's indexes."""
        if self.kind == "median":
            if self.masked and n % 2 and data_dtype.kind == "f":  # numpy.ma.median: (high + high) / 2
                s = np.add(vals[:, 0], vals[:, 0])
                return np.true_divide(s, 2.0, out=s, casting="unsafe")
            return np.mean(vals[:, :1] if n % 2 else vals[:, :2], axis=1)
        idx, vi = self.indexes(int(n), data_dtype)
        exp = np.clip(np.where(idx < 0, n - 1, idx), 0, max(n - 1, 0))
        if not (used == exp).all():
            raise RuntimeError("quantile: the selected ranks differ from NumPy's indexes")
        kq = self.qf.size
        if self._integral():
            return vals[:, :kq]
        prev = idx[:kq].astype(np.intp)
        gamma = fnb._get_gamma(vi, prev, self.props)
        return fnb._lerp(vals[:, :kq], vals[:, kq:], gamma)


# ---- the device selection over this rank's part ---------------------------------------------------------------------------
def _moved_view(src, axis):
    """The IndexView of this rank's part of src with the reduced axis last (every axis: the part as it is)."""
    v = blocks.index_view(src)
    if axis is None:
        return v
    nd = int(v.ndim)
    order = [d for d in range(nd) if d != axis] + [axis]
    shape, stride = [int(v.shape[d]) for d in order], [int(v.stride[d]) for d in order]
    for d in range(nd):
        v.shape[d], v.stride[d] = shape[d], stride[d]
    return v


def _select_rows(view, code, L, S, spec, skip_nan, data_dtype):
    """The `row` form: (keys (S, K) uint64, nans (S,) int64) of this rank's S segments."""
    K = spec.K
    table = spec.ranks(np.arange(L + 1) if skip_nan else np.array([L]), data_dtype)
    d_table = torch.from_numpy(np.ascontiguousarray(table, dtype=np.int64)).to(RT.device)
    keys, nans = _device_i64(S * K), _device_i64(S)
    RT.select_rows(view, code, L, K, d_table.data_ptr(), skip_nan, keys.data_ptr(), nans.data_ptr())
    RT.hold(d_table, keys, nans)
    return keys[:S * K].cpu().numpy().view(np.uint64).reshape(S, K), nans[:S].cpu().numpy()


def _select_passes(view, code, L, S_local, GS, seg_map, spec, skip_nan, data_dtype, reduce):
    """The `pass` form over the GS segments of the whole array: (keys (GS, K), nans (GS,)).  seg_map: None (the view's
    segments are the state's rows) or (local kept shape, global C strides, base row); reduce: sum the counts over the
    ranks."""
    K = spec.K
    f = cabi.group_plan_fields(cabi.describe_select_plan(view, code, L, K, GS))
    digit, passes = f["digit"], f["passes"]
    st = cabi.SelectState()
    st.segments, st.targets = GS, K
    rank, key, slot, slot_key = _device_i64(GS * K), _device_i64(GS * K), _device_i64(GS * K), _device_i64(GS * K)
    n_slots, counts, nans, matched = _device_i64(GS), _device_i64(GS * K << digit), _device_i64(GS), _device_i64(GS)
    cand_n = _device_i64(1, fill=0)
    st.rank, st.key, st.slot, st.slot_key = rank.data_ptr(), key.data_ptr(), slot.data_ptr(), slot_key.data_ptr()
    st.n_slots, st.counts, st.nans, st.matched = n_slots.data_ptr(), counts.data_ptr(), nans.data_ptr(), matched.data_ptr()
    st.cand_n = cand_n.data_ptr()
    if seg_map is not None:
        shape, gst, base = seg_map
        st.seg_dims = len(shape)
        for d, (s, g) in enumerate(zip(shape, gst)):
            st.seg_shape[d], st.seg_gstride[d] = s, g
        st.seg_base = base
    n_total = None
    cand, mode = None, cabi.SELECT_READ
    for p in range(passes):
        RT.select_count(view, code, L, st, p, mode)
        if reduce:
            RT.all_reduce(counts, "sum")
            if p == 0 and data_dtype.kind == "f":
                RT.all_reduce(nans, "sum")
        if p == 0:
            h_nans = nans[:GS].cpu().numpy() if data_dtype.kind == "f" else np.zeros(GS, dtype=np.int64)
            n_total = counts.view(GS, K, -1)[:, 0, :].sum(dim=1).cpu().numpy()  # every key of the segment (row 0)
            nv = n_total - h_nans if skip_nan else n_total
            rank.copy_(torch.from_numpy(np.ascontiguousarray(spec.ranks(nv, data_dtype), dtype=np.int64).reshape(-1)).to(RT.device))
        RT.select_choose(view, code, L, st, p)
        if GS == 1 and mode == cabi.SELECT_READ and p + 2 < passes:
            m = int(matched.cpu()[0])
            cap = builtins.max(int(n_total[0]) // 32, 65536)
            if m <= cap:
                cand = _device_i64(m, fill=0)
                st.cand, st.cand_cap = cand.data_ptr(), builtins.max(m, 1)
                mode = cabi.SELECT_APPEND
        elif mode == cabi.SELECT_APPEND:
            mode = cabi.SELECT_CAND
    RT.hold(rank, key, slot, slot_key, n_slots, counts, nans, matched, cand_n, cand)
    return key[:GS * K].cpu().numpy().view(np.uint64).reshape(GS, K), h_nans


def _finish_all(keys, nans, seg_n, spec, skip_nan, data_dtype, work_dtype):
    """Host results of every segment: shape (S,) + q.shape... as (S, len(q)) or (S,), NumPy's dtype; warns for all-NaN
    slices of a nan variant."""
    S = keys.shape[0]
    vals = values_of(keys, work_dtype).astype(data_dtype)
    nv = seg_n - nans if skip_nan else np.full(S, seg_n, dtype=np.int64) if np.ndim(seg_n) == 0 else seg_n
    nv = np.broadcast_to(np.asarray(nv, dtype=np.int64), (S,))
    out = None
    for n in np.unique(nv):
        sel = np.flatnonzero(nv == n)
        if n == 0:
            continue
        used = spec.ranks(np.array([n]), data_dtype)[0]
        r = spec.finish(vals[sel], int(n), data_dtype, used)
        if out is None:
            out = np.empty((S,) + r.shape[1:], dtype=r.dtype)
        out[sel] = r
    if out is None:  # every slice all-NaN
        out = np.empty((S,) if spec.kind == "median" else (S, spec.qf.size), dtype=data_dtype)
    if data_dtype.kind == "f":
        empty = nv == 0
        if skip_nan and empty.any():
            warnings.warn("All-NaN slice encountered", RuntimeWarning, stacklevel=4)
        bad = empty | (nans > 0) if not skip_nan else empty
        out[bad] = np.nan
    return out


# ---- the public functions -----------------------------------------------------------------------------------------------
def _axis_of(axis, nd):
    if axis is None:
        return None
    if isinstance(axis, (tuple, list)):
        raise NotImplementedError("order statistics over a tuple of axes")
    axis = operator.index(axis)
    if not -builtins.max(nd, 1) <= axis < builtins.max(nd, 1):
        raise np.exceptions.AxisError(axis, nd)
    return axis % builtins.max(nd, 1)


def _host_q(q):
    from . import ramba as R

    return q.asarray() if isinstance(q, R.ndarray) else q


def _numpy_call(name, a, q, **kw):
    return getattr(np, name)(a, q, **kw) if q is not None else getattr(np, name)(a, **kw)


def _wrap(res):
    from . import ramba as R

    return R.fromarray(res) if isinstance(res, np.ndarray) else res


def _order(name, a, q, axis, out, overwrite_input, method, keepdims, weights, interpolation):
    from . import ramba as R

    nan = name.startswith("nan")
    base = name[3:] if nan else name
    kw = {"axis": axis, "out": out, "overwrite_input": overwrite_input}
    if base != "median":
        kw.update(method=method, weights=weights, interpolation=interpolation)
    if keepdims is not np._NoValue:
        kw["keepdims"] = keepdims
    a_nd = R._as_nd(a)
    if not isinstance(a_nd, R.ndarray):
        return _numpy_call(name, a, _host_q(q), **kw)
    a = a_nd
    if out is not None:
        raise NotImplementedError("%s: out= is not supported" % name)
    if weights is not None:
        raise NotImplementedError("%s: weights= is not supported" % name)
    _unmasked(a, name)
    if a.dtype.kind == "c":
        raise TypeError("a must be an array of real numbers")
    if a.dtype not in _HOST_DTYPES:
        raise NotImplementedError("%s of dtype %s" % (name, a.dtype))
    keepdims = bool(keepdims) if keepdims is not np._NoValue else False
    if interpolation is not None:
        method = fnb._check_interpolation_as_method(method, interpolation, name)
    spec = None
    if base != "median":
        qh = _host_q(q)
        if base == "percentile":
            qh = np.true_divide(qh, a.dtype.type(100) if a.dtype.kind == "f" else 100, out=...)
            if not fnb._quantile_is_valid(qh):
                raise ValueError("Percentiles must be in the range [0, 100]")
        else:
            qh = np.asanyarray(qh, dtype=a.dtype) if isinstance(qh, (int, float)) and a.dtype.kind == "f" else np.asanyarray(qh)
            if not fnb._quantile_is_valid(qh):
                raise ValueError("Quantiles must be in the range [0, 1]")
        if qh.ndim > 2:
            raise ValueError("q must be a scalar or 1d")
        if method not in fnb._QuantileMethods:
            raise ValueError("%r is not a valid method. Use one of: %s" % (method, fnb._QuantileMethods.keys()))
        spec = _Spec("quantile", np.asarray(qh), method)
    else:
        spec = _Spec("median")
    if isinstance(axis, (tuple, list)):
        raise NotImplementedError("%s over a tuple of axes" % name)
    if a.size == 0 or a.ndim == 0:  # NumPy's result, exception and warning on a same-dtype stand-in
        stand = np.empty(a.shape, a.dtype) if a.size == 0 else np.asarray(a.asarray(), dtype=a.dtype)
        kw.pop("out")
        kw.pop("weights", None)
        kw.pop("interpolation", None)
        kw["method"] = method if base != "median" else None
        if base == "median":
            kw.pop("method")
        return _wrap(_numpy_call(name, stand, spec.q if spec.q is not None else None, **kw))
    ax = _axis_of(axis, a.ndim)
    if name == "nanmedian" and ax is not None and a.ndim > 1 and a.shape[ax] < 600:
        spec.masked = True  # NumPy's nanmedian takes numpy.ma.median here
    res = _compute(a, ax, spec, nan and a.dtype.kind == "f", keepdims)
    return res


def _compute(a, axis, spec, skip_nan, keepdims):
    from . import ramba as R

    data_dtype = a.dtype
    (src,) = _ready(_source(a))
    work = src.dtype
    code = rb_dtype(work)
    W = common.num_workers
    qshape = () if spec.q is None else spec.q.shape
    kshape = tuple(s for d, s in enumerate(a.shape) if d != axis) if axis is not None else ()
    if axis is None:
        oshape = (1,) * a.ndim if keepdims else ()
    else:
        oshape = tuple(1 if d == axis else s for d, s in enumerate(a.shape)) if keepdims else kshape
    GS = int(np.prod(kshape))
    L = a.size if axis is None else a.shape[axis]
    if W == 1:
        holds, bstart, bsize = True, [0] * a.ndim, list(a.shape)
    else:
        sv = src.distribution[common.worker_num]
        holds = not shardview.is_empty(sv)
        bstart, bsize = [int(x) for x in sv.start], [int(x) for x in sv.size]
    cut = W > 1 and (axis is None or builtins.any(not shardview.is_empty(sv) and (int(sv.start[axis]) != 0 or int(sv.size[axis]) != L)
                                                 for sv in src.distribution))
    if holds:
        view = _moved_view(src, axis)
    else:
        view = cabi.index_view(0, [0], [1], blocks.itemsize(work))
    n_loc = int(np.prod([int(view.shape[d]) for d in range(int(view.ndim))])) if holds else 0
    if not cut:
        S = GS if W == 1 else (int(np.prod([s for d, s in enumerate(bsize) if d != axis])) if holds else 0)
        keys, nans = np.zeros((S, spec.K), np.uint64), np.zeros(S, np.int64)
        if S:
            f = cabi.group_plan_fields(cabi.describe_select_plan(view, code, L, spec.K))
            if f["form"] == "row":
                keys, nans = _select_rows(view, code, L, S, spec, skip_nan, data_dtype)
            else:
                keys, nans = _select_passes(view, code, L, S, S, None, spec, skip_nan, data_dtype, False)
        vals = _finish_all(keys, nans, L, spec, skip_nan, data_dtype, work) if S else None
        if W > 1 and skip_nan:  # every rank warns together
            flag = torch.tensor([int(bool(S) and bool((L - nans == 0).any()))], dtype=torch.int64, device=RT.device)
            RT.all_reduce(flag, "max")
            if int(flag.cpu()[0]) and not (S and (L - nans == 0).any()):
                warnings.warn("All-NaN slice encountered", RuntimeWarning, stacklevel=3)
        if W == 1:
            return _shape_result(vals, qshape, oshape)
        return _local_result(src, vals, qshape, oshape, axis, keepdims, holds, bstart, bsize, data_dtype, spec)
    # every axis at once, or a cut axis: count rows of the global segments, one all-reduce per pass
    if axis is None:
        L_loc, seg_map = builtins.max(n_loc, 1), None
    else:
        L_loc = bsize[axis] if holds and bsize[axis] else 1
        lshape = [s for d, s in enumerate(bsize) if d != axis]
        lstart = [s for d, s in enumerate(bstart) if d != axis]
        gst = _contig_strides(kshape)[0] if kshape else []
        seg_map = (lshape, gst, builtins.sum(s * g for s, g in zip(lstart, gst))) if lshape else None
    keys, nans = _select_passes(view, code, L_loc, None, GS, seg_map, spec, skip_nan, data_dtype, True)
    vals = _finish_all(keys, nans, L, spec, skip_nan, data_dtype, work)
    return _shape_result(vals, qshape, oshape)


def _arrange(vals, qshape, oshape):
    """(S, len(q)) or (S,) host results as NumPy's q.shape + output shape."""
    if vals.ndim == 1:
        return vals.reshape(oshape)
    return np.moveaxis(vals, 1, 0).reshape(qshape + oshape)


def _shape_result(vals, qshape, oshape):
    from . import ramba as R

    r = _arrange(vals, qshape, oshape)
    if r.ndim == 0:  # NumPy's scalar
        return r[()]
    return R.fromarray(np.ascontiguousarray(r))


def _local_result(src, vals, qshape, oshape, axis, keepdims, holds, bstart, bsize, data_dtype, spec):
    """The result partitioned like src over the kept axes (q's axes whole on every rank), each rank writing its block."""
    from . import ramba as R

    nq = len(qshape)
    rdtype = vals.dtype if vals is not None else _result_dtype(spec, data_dtype)
    dist = []
    for sv in src.distribution:
        if shardview.is_empty(sv):
            size, start = [0] * (nq + len(oshape)), [0] * (nq + len(oshape))
        else:
            size = list(qshape) + [1 if d == axis else int(x) for d, x in enumerate(sv.size) if keepdims or d != axis]
            start = [0] * nq + [0 if d == axis else int(x) for d, x in enumerate(sv.start) if keepdims or d != axis]
        dist.append(shardview.shardview(np.array(size, dtype=np.int64), np.array(start, dtype=np.int64)))
    res = R.create_array_with_divisions(qshape + oshape, dist, dtype=rdtype)
    if holds and vals is not None:
        lo = [1 if d == axis else s for d, s in enumerate(bsize) if keepdims or d != axis]
        block = np.ascontiguousarray(_arrange(vals.astype(rdtype), qshape, tuple(lo)))
        sh = blocks.block(res)
        st = _contig_strides(list(block.shape))[0] if block.ndim else [1]
        dev = torch.from_numpy(block.reshape(-1).view(np.uint8).copy()).to(RT.device)
        shape = list(block.shape) if block.ndim else [1]
        c = rb_dtype(rdtype)
        RT.launch(_pack_program(c, c), shape, [0] * len(shape), [(dev.data_ptr(), st, c), (sh.ptr(0), _contig_strides(shape)[0], c, sh.bounds)])
        RT.hold(dev)
    return res


def _result_dtype(spec, data_dtype):
    """NumPy's result dtype for data of data_dtype (a two-element stand-in)."""
    stand = np.zeros(2, data_dtype)
    if spec.kind == "median":
        return np.median(stand).dtype
    return np.asarray(np.quantile(stand, spec.q, method=spec.method)).dtype


def median(a, axis=None, out=None, overwrite_input=False, keepdims=False):
    """NumPy's np.median on the device's order statistics (see the module's docstring for the sign of tied zeros)."""
    return _order("median", a, None, axis, out, overwrite_input, "linear", keepdims, None, None)


def nanmedian(a, axis=None, out=None, overwrite_input=False, keepdims=np._NoValue):
    """NumPy's np.nanmedian: the median of the numbers of each slice; NaN and a RuntimeWarning for an all-NaN slice."""
    return _order("nanmedian", a, None, axis, out, overwrite_input, "linear", keepdims, None, None)


def percentile(a, q, axis=None, out=None, overwrite_input=False, method="linear", keepdims=False, *, weights=None, interpolation=None):
    """NumPy's np.percentile, every method; q a scalar, an array-like or a ramba array (gathered once)."""
    return _order("percentile", a, q, axis, out, overwrite_input, method, keepdims, weights, interpolation)


def nanpercentile(a, q, axis=None, out=None, overwrite_input=False, method="linear", keepdims=np._NoValue, *, weights=None,
                  interpolation=None):
    """NumPy's np.nanpercentile."""
    return _order("nanpercentile", a, q, axis, out, overwrite_input, method, keepdims, weights, interpolation)


def quantile(a, q, axis=None, out=None, overwrite_input=False, method="linear", keepdims=False, *, weights=None, interpolation=None):
    """NumPy's np.quantile, every method."""
    return _order("quantile", a, q, axis, out, overwrite_input, method, keepdims, weights, interpolation)


def nanquantile(a, q, axis=None, out=None, overwrite_input=False, method="linear", keepdims=np._NoValue, *, weights=None,
                interpolation=None):
    """NumPy's np.nanquantile."""
    return _order("nanquantile", a, q, axis, out, overwrite_input, method, keepdims, weights, interpolation)
