"""Integer-array indexing: `a[idx]` and `a[idx] = v` where the index holds lists, integer NumPy arrays or integer ramba
arrays (getitem_array_executor / setitem_array_executor / dim_sizes_from_index, ramba/ramba.py:6429-6545, 6143-6297,
7683-7749).

  * The result shape follows NumPy: the array terms (and the integers among them) broadcast together; the broadcast dims
    take the place of the advanced terms when those are adjacent and go first otherwise.
  * `lin`, the C-order linear index of every addressed element within the source view (-1 where a coordinate is out of
    range), is an ordinary deferred statement over the result's box: slices are iotas, array terms are the index arrays
    broadcast into the box.  Its flush also counts the -1 entries; reading that count synchronises with the device, and
    an out-of-range index raises IndexError before anything is read or written.  At one rank this is the call's only
    synchronisation; at several ranks a second one reads the all-gathered per-owner counts, which size the exchange.
  * One rank: rb200_gather / rb200_scatter on the local view.  Several ranks: rb200_route groups the requests by the
    rank that owns the element; the counts are all-gathered, requests (and, for a write, values) go out in one grouped
    send / receive, owners serve with rb200_gather (or store with rb200_scatter), and a read's replies come back in a
    second grouped exchange and are placed through the slots.  Requests for a rank's own elements never leave its GPU.
These calls run eagerly (they are not recorded in flush scripts); the flushes of lin and of a write's values are
ordinary flushes."""
import builtins
import itertools
import numbers

import numpy as np
import torch

from . import _cabi as cabi
from . import blocks
from . import common
from . import shardview
from .flush import _local_shape
from .program import E, Iota
from .runtime import RT, Shard


def is_advanced_term(t):
    from .ramba import ndarray

    return isinstance(t, list) or (isinstance(t, (np.ndarray, ndarray)) and t.shape != ())


def has_advanced(index):
    return builtins.any(is_advanced_term(t) for t in index)


def _array_term(t):
    """A list / NumPy array / ramba array index term as an integer array (host or ramba); IndexError otherwise."""
    from .ramba import ndarray

    if isinstance(t, ndarray):
        if t.dtype.kind not in "iu":
            raise IndexError("arrays used as indices must be of integer type (got a ramba array of %s)" % t.dtype)
        if t.maskarray is not None:
            raise NotImplementedError("a masked array as an index")
        return t
    a = np.asarray(t)
    if a.dtype == np.bool_:
        raise IndexError("boolean index arrays inside an index are not supported (the result shape would depend on the data)")
    if a.size == 0 and a.dtype.kind == "f":
        a = a.astype(np.int64)  # (an empty list)
    if a.dtype.kind not in "iu":
        raise IndexError("arrays used as indices must be of integer type (got %s)" % a.dtype)
    return a


def _parse(shape, index):
    """(terms, result shape, result position of the broadcast dims).  terms: one (kind, axis, payload) per index entry,
    kind 's' slice (canonical), 'i' integer (wrapped), 'a' array, 'n' newaxis."""
    from .ramba import _slice_len, canonical_dim, canonical_slice

    ndim = len(shape)
    n_spec = builtins.sum(1 for t in index if t is not None and t is not Ellipsis)
    if n_spec > ndim:
        raise IndexError("too many indices for array: array is %d-dimensional, but %d were indexed" % (ndim, n_spec))
    if builtins.sum(1 for t in index if t is Ellipsis) > 1:
        raise IndexError("an index can only have a single ellipsis ('...')")
    terms, axis = [], 0
    for t in index:
        if isinstance(t, np.ndarray) and t.ndim == 0 and t.dtype.kind in "iu":
            t = int(t)
        if t is Ellipsis:
            for _ in range(ndim - n_spec):
                terms.append(("s", axis, slice(0, shape[axis], 1)))
                axis += 1
        elif t is None:
            terms.append(("n", None, None))
        elif isinstance(t, slice):
            terms.append(("s", axis, canonical_slice(t, shape[axis])))
            axis += 1
        elif isinstance(t, (numbers.Integral, np.integer)) and not isinstance(t, (bool, np.bool_)):
            terms.append(("i", axis, canonical_dim(int(t), shape[axis], checkbounds=True, axis=axis)))
            axis += 1
        elif is_advanced_term(t):
            terms.append(("a", axis, _array_term(t)))
            axis += 1
        else:
            raise IndexError("only integers, slices (`:`), ellipsis (`...`), None and integer arrays are valid indices (got %r)" % (t,))
    while axis < ndim:
        terms.append(("s", axis, slice(0, shape[axis], 1)))
        axis += 1
    adv = [j for j, t in enumerate(terms) if t[0] in "ai"]
    bshape = tuple(np.broadcast_shapes(*[t[2].shape for t in terms if t[0] == "a"]))
    adjacent = adv[-1] - adv[0] + 1 == len(adv)
    out, bpos = [], 0 if not adjacent else None
    if not adjacent:
        out.extend(bshape)
    for j, t in enumerate(terms):
        if t[0] == "s":
            terms[j] = t + (len(out),)  # (the result dim it iterates)
            out.append(_slice_len(t[2]))
        elif t[0] == "n":
            out.append(1)
        elif adjacent and j == adv[0]:
            bpos = len(out)
            out.extend(bshape)
    # host index arrays: bounds are checked now; then every value fits in int64 (uint64 is not a dtype the engine stores)
    for j, t in enumerate(terms):
        if t[0] == "a" and isinstance(t[2], np.ndarray):
            _check_bounds(t[2], t[1], shape[t[1]])
            if t[2].dtype not in _STORED_INDEX_DTYPES:
                terms[j] = (t[0], t[1], t[2].astype(np.int64))
    return terms, tuple(out), bpos, bshape


_STORED_INDEX_DTYPES = tuple(np.dtype(d) for d in (np.int64, np.int32, np.int16, np.int8, np.uint32, np.uint16, np.uint8))


def _check_bounds(h, axis, n):
    """IndexError naming the first out-of-range entry of host index array h for an axis of size n."""
    h = np.asarray(h).reshape(-1)
    bad = (h < -n) | (h >= n) if h.dtype.kind == "i" else (h >= n)
    if bad.any():
        raise IndexError("index %d is out of bounds for axis %d with size %d" % (int(h[bad][0]), axis, n))


def _place(arr, rshape, bpos, nb):
    """ramba array `arr` (broadcastable to the broadcast shape of nb dims) as a view of the result's box."""
    k = len(rshape)
    lead = nb - arr.ndim
    axes = list(range(bpos)) + [bpos + d for d in range(lead)] + list(range(bpos + nb, k))
    v = arr.expand_dims(tuple(axes)) if axes else arr
    return v if v.shape == rshape else v.broadcast_to(rshape)


def _lin(src_shape, terms, rshape, bpos, bshape):
    """lin: the C-order linear index within the source of every result element, -1 where a coordinate is out of range."""
    from . import ramba as R

    nb = len(bshape)
    cstr = [1] * len(src_shape)
    for d in range(len(src_shape) - 2, -1, -1):
        cstr[d] = cstr[d + 1] * src_shape[d + 1]
    expr, valid, first = None, None, None
    for t in terms:
        kind, axis, p = t[:3]
        if kind == "n":
            continue
        if kind == "s":
            coord = E("add", p.start, E("mul", p.step, Iota(t[3])))
        elif kind == "i":
            coord = p
        else:
            arr = p if isinstance(p, R.ndarray) else R.fromarray(p)
            if first is None and isinstance(p, R.ndarray):
                first = p
            n = src_shape[axis]
            c = _place(arr, rshape, bpos, nb)
            coord = E("where", E("lt", c, 0), E("add", c, n), c)
            ok = E("land", E("ge", c, -n), E("lt", c, n))
            valid = ok if valid is None else E("land", valid, ok)
        term = coord if cstr[axis] == 1 else E("mul", coord, cstr[axis])
        expr = term if expr is None else E("add", expr, term)
    if expr is None:
        expr = 0
    if valid is not None:
        expr = E("where", valid, expr, -1)
    if first is not None:
        part = _place(first, rshape, bpos, nb)
        lin = R.create_array_with_divisions(rshape, part.distribution, dtype=np.int64)
    else:
        lin = R.empty(rshape, dtype=np.int64)
    R.DAG.assign(lin, expr)
    return lin


def _check_array_terms(src_shape, terms):
    """Raise IndexError for the first out-of-range entry of a ramba index array (copies the index arrays to the host:
    only after the fused count found one, or when the result is empty and no count runs)."""
    for t in terms:
        kind, axis, p = t[:3]
        if kind == "a" and not isinstance(p, np.ndarray) and p.size:
            _check_bounds(p.asarray(), axis, src_shape[axis])


def _route_table(nd):
    """The partition of view nd as a grid: every rank's box, its owner and where the owner keeps it."""
    bd = nd.bdarray
    shape = nd.shape
    boxes = []
    for r, sv in enumerate(nd.distribution):
        if shardview.is_empty(sv):
            continue
        lshape = tuple(int(s) for s in _local_shape(bd.distribution, r))
        strides, _ = Shard.layout(lshape, bd.pad if builtins.all(s > 0 for s in lshape) else 0)
        off, st = RT.bind_view(sv, strides, shardview.clean_range(sv))
        boxes.append((r, [int(x) for x in sv.start], [int(x) for x in sv.size], off, st))
    cuts = []
    for d in range(len(shape)):
        pts = {0, int(shape[d])}
        for (_, st0, sz, _, _) in boxes:
            pts.update((st0[d], st0[d] + sz[d]))
        cuts.append(sorted(pts))
    owners, offsets, strides = [], [], []
    for cell in itertools.product(*[range(len(c) - 1) for c in cuts]):
        lo = [cuts[d][j] for d, j in enumerate(cell)]
        hi = [cuts[d][j + 1] for d, j in enumerate(cell)]
        hit = [b for b in boxes if builtins.all(b[1][d] <= lo[d] and hi[d] <= b[1][d] + b[2][d] for d in range(len(shape)))]
        assert len(hit) == 1, "the partition of an indexed view is not a grid of blocks"
        r, st0, _, off, st = hit[0]
        owners.append(r)
        offsets.append(off + builtins.sum((lo[d] - st0[d]) * st[d] for d in range(len(shape))))
        strides.append(st)
    return cabi.route_table(shape, cuts, owners, offsets, strides, common.num_workers)


def _exchange_counts(counts):
    """counts: this rank's requests per owner (device int64, W entries) -> M[p][q] on the host, for every p."""
    W = common.num_workers
    allc = torch.empty(W * W, dtype=torch.int64, device=RT.device)
    RT.all_gather(allc, counts).wait()
    return allc.cpu().numpy().reshape(W, W)


def _route(nd, lin_ptr, n):
    """Route this rank's n requests on view nd: (offsets, slots, M, starts, keep)."""
    W = common.num_workers
    table, keep = _route_table(nd)
    offs = torch.empty(max(n, 1), dtype=torch.int64, device=RT.device)
    slots = torch.empty(max(n, 1), dtype=torch.int64, device=RT.device)
    counts = torch.zeros(W, dtype=torch.int64, device=RT.device)
    bad = torch.zeros(1, dtype=torch.int64, device=RT.device)
    scratch = RT.route(table, lin_ptr, n, offs.data_ptr(), slots.data_ptr(), counts.data_ptr(), bad.data_ptr())
    M = _exchange_counts(counts)
    mine = M[common.worker_num]
    starts = np.concatenate([[0], np.cumsum(mine)[:-1]]).astype(np.int64)
    return offs, slots, M, starts, [keep, counts, bad, scratch, offs, slots]


def _gather(src, lin_nd, out):
    """out[i] = src[lin[i]] for this rank's block of lin / out."""
    w, W = common.worker_num, common.num_workers
    lin_sh, out_sh = blocks.block(lin_nd), blocks.block(out)
    n = int(np.prod(lin_sh.shape)) if lin_sh.shape else 1
    if shardview.is_empty(lin_nd.distribution[w]):
        n = 0
    bad = torch.zeros(1, dtype=torch.int64, device=RT.device)
    if W == 1:
        RT.gather(blocks.index_view(src), lin_sh.ptr(0), n, out_sh.ptr(0), bad.data_ptr())
        RT.hold(bad)
        return
    isz = blocks.itemsize(src.dtype)
    offs, slots, M, starts, keep = _route(src, lin_sh.ptr(0), n)
    nv = int(M[w].sum())
    flat = blocks.flat_index_view(src)
    rep = torch.empty(max(nv * isz, 1), dtype=torch.uint8, device=RT.device)
    ops, reqs = [], []
    for q in range(W):
        if q != w and M[w][q]:
            ops.append((True, offs[starts[q]:starts[q] + M[w][q]], q))
        if q != w and M[q][w]:
            req = torch.empty(int(M[q][w]), dtype=torch.int64, device=RT.device)
            ops.append((False, req, q))
            reqs.append((q, req))
    for wk in RT.p2p(ops):
        wk.wait()
    if M[w][w]:  # this rank's own elements: straight into the reply buffer
        RT.gather(flat, offs[starts[w]:].data_ptr(), int(M[w][w]), rep[starts[w] * isz:].data_ptr(), bad.data_ptr())
    ops, served = [], []
    for q, req in reqs:
        r = torch.empty(req.numel() * isz, dtype=torch.uint8, device=RT.device)
        RT.gather(flat, req.data_ptr(), req.numel(), r.data_ptr(), bad.data_ptr())
        ops.append((True, r, q))
        served.append(r)
    for q in range(W):
        if q != w and M[w][q]:
            ops.append((False, rep[starts[q] * isz:(starts[q] + M[w][q]) * isz], q))
    for wk in RT.p2p(ops):
        wk.wait()
    if n:
        RT.gather(cabi.index_view(rep.data_ptr(), [nv], [1], isz), slots.data_ptr(), n, out_sh.ptr(0), bad.data_ptr())
    RT.hold(*keep, rep, bad, reqs, served)


def _scatter(dst, lin_nd, vals):
    """dst[lin[i]] = vals[i] for this rank's block of lin / vals."""
    w, W = common.worker_num, common.num_workers
    lin_sh, val_sh = blocks.block(lin_nd), blocks.block(vals)
    n = int(np.prod(lin_sh.shape)) if lin_sh.shape else 1
    if shardview.is_empty(lin_nd.distribution[w]):
        n = 0
    bad = torch.zeros(1, dtype=torch.int64, device=RT.device)
    if W == 1:
        RT.scatter(blocks.index_view(dst), lin_sh.ptr(0), n, val_sh.ptr(0), bad.data_ptr())
        RT.hold(bad)
        return
    isz = blocks.itemsize(dst.dtype)
    offs, slots, M, starts, keep = _route(dst, lin_sh.ptr(0), n)
    nv = int(M[w].sum())
    packed = torch.empty(max(nv * isz, 1), dtype=torch.uint8, device=RT.device)
    if n:  # the values in slot order, grouped by owner
        RT.scatter(cabi.index_view(packed.data_ptr(), [nv], [1], isz), slots.data_ptr(), n, val_sh.ptr(0), bad.data_ptr())
    ops, got = [], []
    for q in range(W):
        if q != w and M[w][q]:
            ops.append((True, offs[starts[q]:starts[q] + M[w][q]], q))
            ops.append((True, packed[starts[q] * isz:(starts[q] + M[w][q]) * isz], q))
        if q != w and M[q][w]:
            req = torch.empty(int(M[q][w]), dtype=torch.int64, device=RT.device)
            v = torch.empty(int(M[q][w]) * isz, dtype=torch.uint8, device=RT.device)
            ops.append((False, req, q))
            ops.append((False, v, q))
            got.append((req, v))
    for wk in RT.p2p(ops):
        wk.wait()
    flat = blocks.flat_index_view(dst)
    if M[w][w]:
        RT.scatter(flat, offs[starts[w]:].data_ptr(), int(M[w][w]), packed[starts[w] * isz:].data_ptr(), bad.data_ptr())
    for req, v in got:
        RT.scatter(flat, req.data_ptr(), req.numel(), v.data_ptr(), bad.data_ptr())
    RT.hold(*keep, packed, bad, got)


def _prepare(a, index):
    if a.maskarray is not None:
        raise NotImplementedError("integer-array indexing of a masked view")
    terms, rshape, bpos, bshape = _parse(a.shape, index)
    return terms, rshape, bpos, bshape


def _address_stream(a, terms, rshape, bpos, bshape):
    """lin for a's elements, after checking every index: raises IndexError if any is out of range."""
    lin = _lin(a.shape, terms, rshape, bpos, bshape)
    if int((lin < 0).astype(np.int64).sum()):
        _check_array_terms(a.shape, terms)
        raise IndexError("index out of bounds")
    return lin


def getitem(a, index):
    """a[index] with at least one integer-array term: a new array (a copy) in a.dtype."""
    from . import ramba as R

    terms, rshape, bpos, bshape = _prepare(a, index)
    size = int(np.prod(rshape)) if rshape else 1
    if size == 0:
        _check_array_terms(a.shape, terms)
        return R.empty(rshape, dtype=a.dtype)
    src = R.copy(a) if common.num_workers > 1 and blocks.overlaps_across_ranks(a) else a
    lin = _address_stream(src, terms, rshape, bpos, bshape)
    out = R.create_array_with_divisions(rshape, lin.distribution, dtype=a.dtype)
    R.DAG.instantiate(src)  # pending writes of the source
    _gather(src, lin, out)
    return out


def setitem(a, index, value):
    """a[index] = value with at least one integer-array term; value converted as in `view[...] = value`."""
    from . import ramba as R

    terms, rshape, bpos, bshape = _prepare(a, index)
    size = int(np.prod(rshape)) if rshape else 1
    if size == 0:
        _check_array_terms(a.shape, terms)
        return
    lin = _address_stream(a, terms, rshape, bpos, bshape)
    vals = R.create_array_with_divisions(rshape, lin.distribution, dtype=a.dtype)
    vals[...] = value
    R.DAG.instantiate(vals)
    R.DAG.before_write(a)
    _scatter(a, lin, vals)
