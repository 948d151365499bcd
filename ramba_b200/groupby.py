"""Grouped reductions along one axis: `a.groupby(dim, labels, num_groups)` (RambaGroupby, ramba/ramba.py:6896-6899,
10185-10643).

  * The labels (one integer per position of axis `dim`) are checked and turned into a CSR table on the host once per
    RambaGroupby: offsets[g] .. offsets[g+1] index the positions of group g, ascending.  The table goes to the device once.
  * sum / prod / min / max / nanmean (NANSUM, NANCOUNT) / var / std (SQDEV against the mean) run rb200_group_reduce on
    this rank's strided view of the source, read in place (slices, steps, transposes, broadcast axes, padded shards).
    count needs no kernel: the per-group counts come from the labels.  The finishing step (cast to the result dtype, the
    division by the counts, the square root) is one fused op per call.
  * Several ranks, two layouts chosen from the partition.  When no rank's block is cut along `dim`, each rank's partial
    is its block of the result, which is partitioned like the source over the kept axes and whole along the group axis:
    nothing is exchanged.  Otherwise every rank reduces its block into a buffer of the result's global shape holding the
    op's identity elsewhere, one all-reduce combines the buffers and every rank keeps its block of the result's default
    distribution: one collective per kernel pass (var and std make two).
  * `gb OP rhs` is `a OP rhs[..., labels, ...]`: the integer-array gather expands rhs along `dim`, then the ordinary
    fused binop runs (an address stream and a gathered array of a's size).
Results are ramba arrays on the GPU.  Differences from the reference: num_groups=None means labels.max() + 1; nanmean
skips NaN; bad labels raise before anything runs; a masked source raises NotImplementedError."""
import builtins

import numpy as np
import torch

from . import _cabi as cabi
from . import blocks
from . import common
from . import shardview
from .flush import _contig_strides, _pack_program
from .program import E, Lowering, np_dtype, rb_dtype, red_identity
from .runtime import RT

_KERNEL_DTYPES = tuple(np.dtype(d) for d in (np.float64, np.float32, np.int64, np.int32))
_ALLREDUCE = {cabi.GROUP_SUM: "sum", cabi.GROUP_PROD: "prod", cabi.GROUP_MIN: "min", cabi.GROUP_MAX: "max",
              cabi.GROUP_NANSUM: "sum", cabi.GROUP_NANCOUNT: "sum", cabi.GROUP_SQDEV: "sum"}


def _int_bounds(dt):
    """(smallest, largest) value of an integer or bool dtype."""
    if dt == np.bool_:
        return 0, 1
    info = np.iinfo(dt)
    return int(info.min), int(info.max)


_finish_programs = {}


def _finish_program(kind, out_code, acc_code):
    """out = acc ("copy"), the divisor ("count"), acc / divisor ("div") or sqrt(acc / divisor) ("sqrt"); views: out, acc,
    divisor (float64)."""
    key = (kind, out_code, acc_code)
    prog = _finish_programs.get(key)
    if prog is None:
        lw = Lowering([out_code, acc_code, cabi.F64])
        if kind == "copy":
            v = lw.read_view(1)
        elif kind in ("min", "max"):  # an empty group's int64 identity becomes the bound of a narrower integer dtype
            lo, hi = _int_bounds(np_dtype(out_code))
            v = lw.build(E(kind, lw.read_view(1), lw.scalar(hi if kind == "min" else lo)), None)
        elif kind == "count":
            v = lw.read_view(2)
        else:
            v = lw.build(E("div", lw.read_view(1), lw.read_view(2)), None)
            if kind == "sqrt":
                v = lw.build(E("sqrt", v), None)
        lw.store(0, v)
        prog = _finish_programs[key] = lw.finish()
    return prog


class _Acc:
    """The accumulators of one kernel pass, readable at any box of the result that this rank can see: its own block (the
    axis is not cut) or the whole all-reduced result (it is).  It owns every device buffer of the pass (`keep`: the
    kernel's scratch and local output).  Buffers are released only after the launches that use them have been enqueued on
    the current stream, where the allocator hands them out again in stream order."""

    __slots__ = ("buf", "origin", "strides", "code", "keep")

    def __init__(self, buf, origin, strides, code, keep=()):
        self.buf, self.origin, self.strides, self.code, self.keep = buf, origin, strides, code, keep

    def at(self, start):
        off = builtins.sum((int(s) - int(o)) * st for s, o, st in zip(start, self.origin, self.strides))
        return self.buf.data_ptr() + off * self.buf.element_size()


class RambaGroupby:
    """`array_to_group` grouped along axis `dim` by `group_array` (host int64 labels) into `num_groups` groups."""

    def __init__(self, array_to_group, dim, group_array, num_groups=None):
        from .ramba import ndarray

        a = array_to_group
        if a.maskarray is not None:
            raise NotImplementedError("groupby of a masked array")
        if a.ndim == 0:
            raise ValueError("groupby needs an array with at least one dimension")
        if not isinstance(dim, (int, np.integer)) or isinstance(dim, (bool, np.bool_)) or not -a.ndim <= int(dim) < a.ndim:
            raise ValueError("groupby: dim %r is not an axis of a %d-d array" % (dim, a.ndim))
        dim = int(dim) % a.ndim
        labels = group_array.asarray() if isinstance(group_array, ndarray) else np.asarray(group_array)
        if labels.ndim != 1 or labels.shape[0] != a.shape[dim]:
            raise ValueError("groupby: the labels must be a 1-d array of length %d (the extent of axis %d), got shape %s"
                             % (a.shape[dim], dim, labels.shape))
        if labels.size == 0 and labels.dtype.kind == "f":
            labels = labels.astype(np.int64)
        if labels.dtype.kind not in "iu":
            raise ValueError("groupby: labels must be integers (got %s)" % labels.dtype)
        if labels.dtype.kind == "u" and labels.size and int(labels.max()) > np.iinfo(np.int64).max:
            raise IndexError("groupby: label %d is out of range" % int(labels.max()))
        labels = labels.astype(np.int64)
        if num_groups is None:
            if labels.size == 0:
                raise ValueError("groupby: num_groups=None needs at least one label")
            num_groups = int(labels.max()) + 1
        if not isinstance(num_groups, (int, np.integer)) or int(num_groups) < 1 or int(num_groups) >= 2 ** 31:
            raise ValueError("groupby: num_groups must be an integer in [1, 2**31), got %r" % (num_groups,))
        G = int(num_groups)
        bad = (labels < 0) | (labels >= G)
        if bad.any():
            raise IndexError("groupby: label %d at position %d is outside [0, %d)" % (int(labels[bad][0]), int(np.argmax(bad)), G))
        self.array_to_group = a
        self.dim = dim
        self.group_array = labels
        self.num_groups = G
        self._counts = np.bincount(labels, minlength=G).astype(np.int64)
        self._members = np.argsort(labels, kind="stable").astype(np.int64)
        self._offsets = np.concatenate([[0], np.cumsum(self._counts)]).astype(np.int64)
        self._tables = {}  # (first position, length) of an axis segment -> (GroupTable, device arrays)
        self._counts_dev = None

    # ---- the CSR table of an axis segment, on the device
    def _table(self, s0, n):
        hit = self._tables.get((s0, n))
        if hit is None:
            if s0 == 0 and n == len(self.group_array):
                offs, mem = self._offsets, self._members
            else:
                seg = self.group_array[s0:s0 + n]
                cnt = np.bincount(seg, minlength=self.num_groups)
                offs = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
                mem = np.argsort(seg, kind="stable").astype(np.int64)
            d_offs = torch.from_numpy(offs).to(RT.device)
            d_mem = torch.from_numpy(mem if len(mem) else np.zeros(1, np.int64)).to(RT.device)
            hit = self._tables[(s0, n)] = (cabi.group_table(self.num_groups, n, d_offs.data_ptr(), d_mem.data_ptr()), (d_offs, d_mem))
        return hit[0]

    def _counts_device(self):
        if self._counts_dev is None:
            self._counts_dev = torch.from_numpy(self._counts.astype(np.float64)).to(RT.device)
        return self._counts_dev

    # ---- source and layout
    def _source(self):
        from . import ramba as R

        a = self.array_to_group
        if a.dtype not in _KERNEL_DTYPES:  # bool and small integers: one fused widening copy
            a = a.astype(np.float64 if a.dtype.kind == "f" else np.int64)
        if common.num_workers > 1 and blocks.overlaps_across_ranks(a):  # broadcast views overlap between ranks
            a = R.copy(a)
        R.DAG.instantiate(a)
        return a

    def _rshape(self, shape):
        s = list(shape)
        s[self.dim] = self.num_groups
        return tuple(s)

    def _axis_cut(self, src):
        ax, L = self.dim, src.shape[self.dim]
        if L == 0:
            return True
        return builtins.any(not shardview.is_empty(sv) and (int(sv.start[ax]) != 0 or int(sv.size[ax]) != L) for sv in src.distribution)

    def _pass(self, src, op, cut, center=None):
        """One rb200_group_reduce of this rank's view (+ the all-reduce when the axis is cut) -> _Acc."""
        w = common.worker_num
        ax, G = self.dim, self.num_groups
        is_f = src.dtype.kind == "f" or op == cabi.GROUP_SQDEV
        tdt = torch.float64 if is_f else torch.int64
        code = cabi.F64 if is_f else cabi.I64
        ident = red_identity(_ALLREDUCE[op], np.float64 if is_f else np.int64)
        bstart, bsize = self._block(src)
        mine = self._holds_block(src)
        lstart = list(bstart)
        lstart[ax] = 0
        lshape = self._rshape(bsize)
        n_loc = int(np.prod(lshape)) if mine else 0
        local = torch.empty(max(n_loc, 1), dtype=tdt, device=RT.device)
        scratch = None
        if mine and bsize[ax] == 0:  # an empty grouped axis: every group is empty
            local.fill_(ident)
        elif mine:
            view = blocks.index_view(src)
            table = self._table(bstart[ax], bsize[ax])
            scratch = RT.group_reduce(view, rb_dtype(src.dtype), ax, table, op, center, local.data_ptr())
        if not cut:
            return _Acc(local, lstart, _contig_strides(lshape)[0], code, (scratch,))
        rshape = self._rshape(src.shape)
        glob = torch.full((max(int(np.prod(rshape)), 1),), ident, dtype=tdt, device=RT.device)
        gst = _contig_strides(rshape)[0]
        if n_loc:
            off = builtins.sum(s * st for s, st in zip(lstart, gst))
            RT.launch(_pack_program(code, code), lshape, [0] * len(lshape),
                      [(local.data_ptr(), _contig_strides(lshape)[0], code), (glob.data_ptr() + off * 8, gst, code)])
        RT.all_reduce(glob, _ALLREDUCE[op])
        return _Acc(glob, [0] * len(rshape), gst, code, (local, scratch))

    def _center(self, src, acc):
        """The group means in the layout of this rank's kernel output (float64, contiguous), for SQDEV."""
        if not self._holds_block(src):
            return None
        start, size = self._block(src)
        start[self.dim] = 0
        shape = self._rshape(size)
        buf = torch.empty(max(int(np.prod(shape)), 1), dtype=torch.float64, device=RT.device)
        self._launch_finish("div", buf.data_ptr(), cabi.F64, None, shape, acc, start, self._count_view(start))
        return buf

    @staticmethod
    def _block(src):
        """(start, size) of this rank's part of the source (at one rank: the whole source, also when it is empty)."""
        if common.num_workers == 1:
            return [0] * src.ndim, [int(x) for x in src.shape]
        sv = src.distribution[common.worker_num]
        return [int(x) for x in sv.start], [int(x) for x in sv.size]

    def _holds_block(self, src):
        """Whether this rank computes a block of the result: its part of the source is not empty (at one rank: the
        result is not empty, even when the grouped axis is)."""
        if common.num_workers == 1:
            return builtins.all(int(s) > 0 for d, s in enumerate(src.shape) if d != self.dim)
        return not shardview.is_empty(src.distribution[common.worker_num])

    def _count_view(self, start):
        st = [0] * self.array_to_group.ndim
        st[self.dim] = 1
        return self._counts_device().data_ptr() + int(start[self.dim]) * 8, st

    def _launch_finish(self, kind, out_ptr, out_code, out_bounds, shape, acc, start, div):
        if int(np.prod(shape)) == 0:
            return
        prog = _finish_program(kind, out_code, acc.code if acc is not None else cabi.F64)
        acc_ptr, acc_st = (acc.at(start), acc.strides) if acc is not None else (div[0], div[1])
        RT.launch(prog, list(shape), [0] * len(shape),
                  [(out_ptr, _contig_strides(shape)[0], out_code, out_bounds), (acc_ptr, acc_st, acc.code if acc is not None else cabi.F64),
                   (div[0], div[1], cabi.F64)])

    def _result(self, src, cut, dtype):
        """The result array and this rank's block of it: (array, start, shape, shard)."""
        from . import ramba as R

        rshape = self._rshape(src.shape)
        if cut or common.num_workers == 1:
            res = R.empty(rshape, dtype=dtype)
        else:
            ax = self.dim
            dist = []
            for sv in src.distribution:
                size = [int(x) for x in sv.size]
                start = [int(x) for x in sv.start]
                if not shardview.is_empty(sv):
                    size[ax], start[ax] = self.num_groups, 0
                dist.append(shardview.shardview(np.array(size, dtype=np.int64), np.array(start, dtype=np.int64)))
            res = R.create_array_with_divisions(rshape, dist, dtype=dtype)
        sh = blocks.block(res)
        sv = res.distribution[common.worker_num]
        start = [int(x) for x in sv.start]
        shape = [int(x) for x in sv.size] if not shardview.is_empty(sv) else [0] * len(rshape)
        return res, start, shape, sh

    def _aggregate(self, what):
        src = self._source()
        cut = common.num_workers > 1 and self._axis_cut(src)
        a_dt = self.array_to_group.dtype
        f64 = np.dtype(np.float64)
        if what == "count":
            res, start, shape, sh = self._result(src, cut, np.int64)
            self._launch_finish("count", sh.ptr(0), cabi.I64, sh.bounds, shape, None, start, self._count_view(start))
            return res
        if what in ("sum", "prod", "min", "max"):
            op = {"sum": cabi.GROUP_SUM, "prod": cabi.GROUP_PROD, "min": cabi.GROUP_MIN, "max": cabi.GROUP_MAX}[what]
            acc = self._pass(src, op, cut)
            res, start, shape, sh = self._result(src, cut, a_dt)
            narrow_int = a_dt.kind in "iub" and a_dt.itemsize < 8
            kind = what if what in ("min", "max") and narrow_int else "copy"
            self._launch_finish(kind, sh.ptr(0), rb_dtype(a_dt), sh.bounds, shape, acc, start, self._count_view(start))
            return res
        if what == "nanmean":
            acc = self._pass(src, cabi.GROUP_NANSUM, cut)
            cnt = self._pass(src, cabi.GROUP_NANCOUNT, cut) if src.dtype.kind == "f" else None  # (integers: the group size)
            res, start, shape, sh = self._result(src, cut, f64)
            div = (cnt.at(start), cnt.strides) if cnt is not None else self._count_view(start)
            self._launch_finish("div", sh.ptr(0), cabi.F64, sh.bounds, shape, acc, start, div)
            return res
        acc = self._pass(src, cabi.GROUP_SUM, cut)
        if what == "mean":
            res, start, shape, sh = self._result(src, cut, f64)
            self._launch_finish("div", sh.ptr(0), cabi.F64, sh.bounds, shape, acc, start, self._count_view(start))
            return res
        center = self._center(src, acc)
        sq = self._pass(src, cabi.GROUP_SQDEV, cut, center.data_ptr() if center is not None else None)
        res, start, shape, sh = self._result(src, cut, f64)
        self._launch_finish("div" if what == "var" else "sqrt", sh.ptr(0), cabi.F64, sh.bounds, shape, sq, start, self._count_view(start))
        return res

    # ---- aggregations (`dim` is accepted and ignored, as in the reference)
    def sum(self, dim=None):
        return self._aggregate("sum")

    def prod(self, dim=None):
        return self._aggregate("prod")

    def min(self, dim=None):
        return self._aggregate("min")

    def max(self, dim=None):
        return self._aggregate("max")

    def count(self, dim=None):
        return self._aggregate("count")

    def mean(self, dim=None):
        return self._aggregate("mean")

    def nanmean(self, dim=None):
        return self._aggregate("nanmean")

    def var(self, dim=None):
        return self._aggregate("var")

    def std(self, dim=None):
        return self._aggregate("std")

    # ---- a OP rhs[..., labels, ...]
    def _expand(self, rhs):
        from . import ramba as R

        r = rhs if isinstance(rhs, R.ndarray) else R.fromarray(np.asarray(rhs))
        want = self._rshape(self.array_to_group.shape)
        if tuple(r.shape) != want:
            raise ValueError("groupby binop: the right operand must have the aggregate's shape %s, got %s" % (want, tuple(r.shape)))
        return r[(slice(None),) * self.dim + (self.group_array,)]

    def _binop(self, name, rhs):
        return getattr(self.array_to_group, name)(self._expand(rhs))


def _make(name):
    def _method(self, rhs):
        return self._binop(name, rhs)

    _method.__name__ = name
    return _method


def _install_binops(names):
    for n in names:
        setattr(RambaGroupby, n, _make(n))


def groupby(a, dim, value_to_group, num_groups=None):
    return RambaGroupby(a, dim, value_to_group, num_groups)
