"""ramba_b200.flush — this rank's share of one flush (RemoteState.run_deferred_ops, ramba/ramba.py:3493-3819).

run_deferred_ops allocates the shards a fused op touches on first use and runs the flush's script.  The first flush with
a given key plans that script (_plan, recorded on a _FlushTape) without launching or transferring anything: it
classifies every operand view as local / partly remote (is_compat / get_overlaps / intersect,
ramba/ramba.py:3558-3644), brings the remote pieces through the runtime's transfers (halo pieces by one grouped send /
receive, operands every rank needs whole by one all-gather), cuts the iteration box into ranges in which every operand
has exactly one source (get_range_splits_list, ramba/ramba.py:3698-3706) and launches the op list once per range.  One
runner (_replay_tape) executes every flush, the first with its key as well as the later ones.

The helpers the array code shares with it (_local_shape, _pack_program, _combine_program, _contig_strides) live here
too.  Everything a flush needs is handed to it (the view table holds each operand's bdarray), so this module depends on
the runtime and the partition algebra only, never on the array API in ramba.py.
"""
import builtins
import copy
import ctypes

import numpy as np
import torch

from . import _cabi as cabi
from . import common
from . import shardview
from .program import REDUCTIONS, Lowering, ProgramError, fold_expr, rb_dtype
from .runtime import RT, _VERIFY_PLAN_CACHE, fill_template, torch_dtype


_pack_programs = {}


def _pack_program(src_code, dst_code):
    key = (src_code, dst_code)
    if key not in _pack_programs:
        lw = Lowering([src_code, dst_code])
        lw.store(1, lw.read_view(0))
        _pack_programs[key] = lw.finish()
    return _pack_programs[key]


_combine_programs = {}


def _combine_program(red_code, acc_code, combine):
    """red_view = red_view (combine) partial  — applies stage-1 axis partials to the partial array."""
    key = (red_code, acc_code, combine)
    if key not in _combine_programs:
        lw = Lowering([red_code, acc_code])
        tv = lw.build(fold_expr(combine, lw.read_view(0), lw.read_view(1)), None)
        lw.store(0, tv)
        _combine_programs[key] = lw.finish()
    return _combine_programs[key]


def _local_shape(bd_dist, w):
    sv = bd_dist[w]
    return tuple(int(x) for x in sv.size)


def _contig_strides(shape, bcast=None):
    """(C-order element strides of `shape`, 0 along the dims where bcast is true; element count)."""
    st = [0] * len(shape)
    acc = 1
    for d in reversed(range(len(shape))):
        if bcast is not None and bcast[d]:
            st[d] = 0
        else:
            st[d] = acc
            acc *= int(shape[d])
    return st, acc


def _gatherable(vd, exec_dist, bc, vshape, W):
    """Elements per rank if view distribution `vd` can be brought to every rank with one all-gather: every rank runs a
    non-empty part of the iteration box, no rank holds what it needs, every rank needs every rank's WHOLE part, and the
    parts are equal consecutive chunks along the outermost non-broadcast axis (so that rank order == C order).  All
    ranks evaluate this on the same metadata, so they agree.  None otherwise."""
    k = len(bc)
    nb = [d for d in range(k) if not bc[d] and int(vshape[d]) > 1]
    if not nb:
        return None
    a = nb[0]
    m = None
    for p in range(W):
        part = vd[p]
        ex = shardview.clean_range(exec_dist[p])
        if shardview.is_empty(part) or shardview.is_empty(ex) or shardview.is_compat(ex, part):
            return None
        if builtins.any((int(part.axis_map[d]) < 0) != bc[d] for d in range(k)):
            return None
        for d in range(k):
            if bc[d]:
                continue
            if d == a:
                if m is None:
                    m = int(part.size[d])
                if int(part.size[d]) != m or int(part.start[d]) != p * m:
                    return None
            elif int(part.start[d]) != 0 or int(part.size[d]) != int(vshape[d]):
                return None
    # every rank's box must cover the whole operand along its non-broadcast axes
    for j in range(W):
        ex = shardview.clean_range(exec_dist[j])
        for d in range(k):
            if not bc[d] and (int(ex.start[d]) != 0 or int(ex.size[d]) != int(vshape[d])):
                return None
    n = m
    for d in nb[1:]:
        n *= int(vshape[d])
    if m * W != int(vshape[a]) or n * W > (1 << 22):
        return None
    return n


def _ring_receivable(bd_dist, vd, exec_dist, w, W, shard):
    """True when every remote piece of view distribution `vd` this rank needs lies within `shard.border` elements of its
    own block (in every dim), i.e. can be received into the ring of the padded block and then be addressed by this
    rank's own shardview of the view, extended past its box (what LocalNdarray.getborder prepares,
    ramba/ramba.py:1260-1322, regions from shardview.compute_from_border, ramba/shardview_array.py:1069-1136)."""
    mine = vd[w]
    if shardview.is_empty(mine):
        return False
    k = len(mine.size)
    b = shard.border
    for d in range(k):
        if int(mine.axis_map[d]) < 0 or int(mine.steps[d]) < 1:
            return False
    for peer in range(W):
        if peer == w:
            continue
        part = shardview.intersect(vd[peer], exec_dist[w])
        if shardview.is_empty(part):
            continue
        theirs = vd[peer]
        for d in range(k):
            a = int(mine.axis_map[d])
            st = int(mine.steps[d])
            if int(theirs.axis_map[d]) != a or int(theirs.steps[d]) != st:
                return False
            lo = int(mine.base_offset[a]) + (int(part.start[d]) - int(mine.start[d])) * st  # my block coordinates
            hi = lo + (int(part.size[d]) - 1) * st
            if lo < -b or hi > shard.shape[a] - 1 + b:
                return False
            # the same element through the owner's addressing: both must name the same global coordinate
            g_theirs = int(bd_dist[peer].start[a]) + int(theirs.base_offset[a]) + (int(part.start[d]) - int(theirs.start[d])) * st
            if int(bd_dist[w].start[a]) + lo != g_theirs:
                return False
    return True


_plan_cache = {}  # flush key -> script (_FlushTape.finish)


class _FlushTape:
    """The script of one flush, recorded by _plan without launching or transferring anything: buffer allocations, launches
    (the bound rb200_fused_op with its pointers replaced by (resource, byte offset) pairs: a resource is the shard of one
    of the flush's views or one of the buffers the script allocates), the all-gather, the grouped sends / receives, the
    points where the launching stream waits for them, the fold of axis partials.  The buffers are real only so that
    _resolve can name the addresses bound into a launch; nothing is enqueued on them, and they die with the planner."""

    def __init__(self, shards):
        self.shards = shards
        self.actions = []
        self.buffers = []
        self.ring_receives = 0  # halo pieces received into the ring of a padded block (a placement, not a transfer)
        self.in_flight = False  # transfers recorded and not yet waited for

    # ---- resources
    def _resolve(self, p):
        """Device address -> (0, view index, byte offset from the start of that shard's buffer) | (1, buffer slot, offset)."""
        if not p:
            return None
        for i, sh in enumerate(self.shards):
            lo, hi = sh.bounds
            if lo <= p < hi:
                return (0, i, p - lo)
        for k, b in enumerate(self.buffers):
            lo = b.data_ptr()
            if lo <= p < lo + builtins.max(1, b.numel() * b.element_size()):
                return (1, k, p - lo)
        if p == RT.red_scratch().data_ptr():
            return (2, 0, 0)
        raise ProgramError("internal: a bound pointer belongs to no shard or buffer of this flush")

    def empty(self, n, dtype):
        t = torch.empty(n, dtype=dtype, device=RT.device)
        self.actions.append(("alloc", int(n), dtype))
        self.buffers.append(t)
        return t

    def launch(self, *args, **kw):
        fop = RT.bind(*args, **kw)
        patches = []
        for v in range(fop.n_views):
            one = fop.views[v]
            patches.append((self._resolve(one.base), one.alloc_lo is not None and one.alloc_lo != 0))
            one.base = 0
            one.alloc_lo = 0
            one.alloc_hi = 0
        rp = []
        for sl in range(fop.n_reds):
            rp.append(self._resolve(fop.reds[sl].out))
            fop.reds[sl].out = 0
        scratch = self._resolve(fop.red_scratch)
        fop.red_scratch = 0
        self.actions.append(("launch", ctypes.string_at(ctypes.addressof(fop), ctypes.sizeof(fop)), tuple(patches), tuple(rp), scratch))

    def all_gather(self, full, mine):
        self.actions.append(("allgather", self._slot(full), self._slot(mine)))
        self.in_flight = True

    def _slot(self, t):
        for k, b in enumerate(self.buffers):
            if b is t:
                return k
        raise ProgramError("internal: a transfer buffer the flush did not allocate")

    def p2p(self, ops):
        """ops: [(is_send, buffer, peer)], sent / received by ONE grouped launch."""
        self.actions.append(("p2p", tuple([(bool(s), self._slot(b), int(peer)) for (s, b, peer) in ops])))
        self.in_flight = True

    def wait(self):
        """The launching stream waits for the transfers in flight; the host does not."""
        if self.in_flight:
            self.actions.append(("wait",))
            self.in_flight = False

    def reduce_partials(self, out_ptr, in_ptr, n, k, stride_k, code, rop):
        self.actions.append(("fold", self._resolve(out_ptr), self._resolve(in_ptr), int(n), int(k), int(stride_k), int(code), int(rop)))

    def finish(self):
        return (tuple(self.actions), self.ring_receives)


def _addr(res, shards, bufs):
    kind, idx, off = res
    if kind == 0:
        return shards[idx].bounds[0] + off
    if kind == 1:
        return bufs[idx].data_ptr() + off
    return RT.red_scratch().data_ptr()


def _replay_tape(script, shards):
    """Execute a flush script (_FlushTape) against this flush's shards: the one code that runs a flush."""
    actions, ring_receives = script
    bufs = []
    works = []
    for a in actions:
        k = a[0]
        if k == "launch":
            _, template, patches, rp, scratch = a
            views = [(_addr(res, shards, bufs), shards[res[1]].bounds if bounded else None) for res, bounded in patches]
            outs = [None if res is None else _addr(res, shards, bufs) for res in rp]
            RT.submit(fill_template(template, views, outs, None if scratch is None else _addr(scratch, shards, bufs)))
        elif k == "alloc":
            bufs.append(torch.empty(a[1], dtype=a[2], device=RT.device))
        elif k == "p2p":
            works += RT.p2p([(s, bufs[b], peer) for (s, b, peer) in a[1]])
        elif k == "wait":
            for wk in works:
                wk.wait()
            works = []
        elif k == "allgather":
            works.append(RT.all_gather(bufs[a[1]], bufs[a[2]]))
        else:  # fold
            RT.reduce_partials(_addr(a[1], shards, bufs), _addr(a[2], shards, bufs), a[3], a[4], a[5], a[6], a[7])
    for wk in works:
        wk.wait()
    RT.ring_receives += ring_receives
    # staging buffers are torch allocations consumed on the launching stream: the caching allocator reuses them in
    # stream order, so no host synchronisation is needed here
    RT.hold(*bufs)


def run_deferred_ops(views, prog, exec_dist, gred, ared, red_axes):
    """This worker's share of one flush (RemoteState.run_deferred_ops, ramba/ramba.py:3493-3819).  views: the fuser's
    view table, (gid, operand) pairs; an operand has the view's shape, dtype and distribution and its bdarray as `bd`."""
    w, W = common.worker_num, common.num_workers
    # allocate shards on first touch
    shards = []
    for (gid, det) in views:
        bd = det.bd
        sh = RT.shards.get(gid)
        if sh is None:
            sh = RT.create_array(gid, _local_shape(bd.distribution, w), bd.dtype, bd.pad)
        shards.append(sh)
    # ---- flush memo: apart from the buffer addresses, everything a flush does is a function of (op list, partitions of
    # the op and of every operand, shard layouts).  A flush is planned into a script of allocations / launches /
    # transfers / waits with symbolic addresses (_plan) once per key; every flush runs its key's script.
    pkey = (prog, w, W, tuple([sv.key() for sv in exec_dist]), tuple([tuple([sv.key() for sv in det.distribution]) for (_, det) in views]),
            tuple([(sh.shape, sh.border) for sh in shards]), tuple(red_axes) if red_axes else (),
            # (what the ring of a padded block can receive depends on the partition of the whole array)
            tuple([tuple([sv.key() for sv in det.bd.distribution]) if sh.border else None
                   for (_, det), sh in zip(views, shards)]) if W > 1 else ())
    script = _plan_cache.get(pkey)
    if script is None or _VERIFY_PLAN_CACHE:
        planned = _plan(views, shards, prog, exec_dist, gred, ared, red_axes)
        if script is None:
            if len(_plan_cache) >= 1024:
                _plan_cache.clear()
            _plan_cache[pkey] = planned
        elif planned != script:
            raise AssertionError("flush-script memo: planning the same flush again gives a different script")
        script = planned
    _replay_tape(script, shards)


class _Source:
    """An operand's source over iteration box `box`: this rank's block `shard` through shardview `sv`, or the staging
    buffer `buf` holding the box with element strides `cst`.  `received`: a range that reads it waits for the transfers."""

    def __init__(self, box, code, shard=None, sv=None, buf=None, cst=None, received=False):
        self.box, self.code, self.shard, self.sv, self.buf, self.cst, self.received = box, code, shard, sv, buf, cst, received

    def bind(self, r):
        """This source over range r (inside its box), as a bound view of RT.bind."""
        if self.sv is not None:
            off, st = RT.bind_view(self.sv, self.shard.strides, r)
            return (self.shard.ptr(off), st, self.code, self.shard.bounds)
        off = 0
        for d in range(len(self.cst)):
            off += int(r.start[d] - self.box.start[d]) * self.cst[d]
        return (self.buf.data_ptr() + off * self.buf.element_size(), list(self.cst), self.code)


def _packed(part, bc):
    """(shape, element strides, element count) of box `part` of a view packed in C order, broadcast dims collapsed."""
    shp = [1 if bc[d] else int(part.size[d]) for d in range(len(bc))]
    cst, n = _contig_strides(shp, bc)
    return shp, cst, n


def _view_index(views, red_view):
    return [j for j, (g, det) in enumerate(views) if g == red_view.gid and shardview.dist_is_eq(det.distribution, red_view.distribution)][0]


def _plan(views, shards, prog, exec_dist, gred, ared, red_axes):
    """The script (_FlushTape) of this rank's share of one flush.  Launches and transfers nothing."""
    w, W = common.worker_num, common.num_workers
    subspace = shardview.clean_range(exec_dist[w])
    nviews = len(views)
    vdist = [det.distribution for (_, det) in views]
    tape = _FlushTape(shards)
    vcode = [rb_dtype(det.dtype) for (_, det) in views]
    written = [bool(prog.view_written.get(i)) for i in range(nviews)]
    # which views are aligned with the iteration box on every worker?
    local_everywhere = []
    clean_exec = [shardview.clean_range(exec_dist[j]) for j in range(W)]
    for i in range(nviews):
        ok = True
        if vdist[i] is not exec_dist:  # (the common case: the operand's distribution IS the op's)
            for j in range(W):
                ss = clean_exec[j]
                if shardview.is_empty(ss):
                    continue
                if not shardview.is_compat(ss, vdist[i][j]):
                    ok = False
                    break
        local_everywhere.append(ok)

    def copy_part(i, part, bc, buf, unpack=False):
        """Launch arguments of the copy between box `part` of this rank's block of view i and the contiguous buffer
        `buf` (_packed): block -> buffer, or buffer -> block when unpack."""
        shp, cst, _ = _packed(part, bc)
        off, st = RT.bind_view(vdist[i][w], shards[i].strides, part)
        block = (shards[i].ptr(off), [0 if bc[d] else st[d] for d in range(len(bc))], vcode[i])
        flat = (buf.data_ptr(), cst, vcode[i])
        return _pack_program(vcode[i], vcode[i]), shp, [0] * len(shp), [flat, block] if unpack else [block, flat]

    parts = [[] for _ in range(nviews)]  # parts[i]: the _Sources of view i
    gathered = set()         # views served whole by an all-gathered buffer
    ring = [False] * nviews  # views whose remote pieces are received into the ring of this rank's padded block
    post_wait = []           # unpack launches that need the received data (copy_part's launch arguments)
    if W > 1 and not builtins.all(local_everywhere):
        ops = []
        for i in range(nviews):
            if local_everywhere[i]:
                continue
            if written[i]:
                raise ProgramError("fused op writes a view that is not aligned with its iteration space")
            bc = [int(a) < 0 for a in vdist[i][0].axis_map]
            ring[i] = shards[i].border > 0 and not shardview.is_empty(subspace) and _ring_receivable(
                views[i][1].bd.distribution, vdist[i], exec_dist, w, W, shards[i])
            tdt = torch_dtype(views[i][1].dtype)
            g = _gatherable(vdist[i], exec_dist, bc, views[i][1].shape, W)
            if g is not None:
                # every rank needs every rank's part of this (small) operand and the parts are equal consecutive
                # chunks: ONE all-gather into a buffer that then serves the whole iteration box as a single source
                # (the reference ships W*(W-1) pickled pieces, ramba/ramba.py:3646-3693)
                mine = tape.empty(g, tdt)
                tape.launch(*copy_part(i, shardview.clean_range(vdist[i][w]), bc, mine))
                full = tape.empty(W * g, tdt)
                tape.all_gather(full, mine)
                vshape = views[i][1].shape
                fshape = [1 if bc[d] else int(vshape[d]) for d in range(len(bc))]
                fst, _ = _contig_strides(fshape, bc)
                box = shardview.ShardView(np.array([int(subspace.size[d]) if bc[d] else int(vshape[d]) for d in range(len(bc))], dtype=np.int64),
                                          np.array([int(subspace.start[d]) if bc[d] else 0 for d in range(len(bc))], dtype=np.int64))
                parts[i].append(_Source(box, vcode[i], buf=full, cst=fst, received=True))
                gathered.add(i)
                continue
            for peer in range(W):
                if peer == w:
                    continue
                # what `peer` needs from me
                pe = shardview.clean_range(exec_dist[peer])
                if not shardview.is_empty(pe) and not shardview.is_compat(pe, vdist[i][peer]):
                    part = shardview.intersect(vdist[i][w], exec_dist[peer])
                    if not shardview.is_empty(part):
                        buf = tape.empty(max(_packed(part, bc)[2], 1), tdt)
                        tape.launch(*copy_part(i, part, bc, buf))
                        ops.append((True, buf, peer))
                # what I need from `peer`
                if not shardview.is_empty(subspace) and not shardview.is_compat(subspace, vdist[i][w]):
                    part = shardview.intersect(vdist[i][peer], exec_dist[w])
                    if not shardview.is_empty(part):
                        _, cst, n = _packed(part, bc)
                        buf = tape.empty(max(n, 1), tdt)
                        ops.append((False, buf, peer))
                        pb = shardview.clean_range(part)
                        if ring[i]:
                            # getborder (ramba/ramba.py:1260-1322): the neighbour's edge lands in the ring of MY padded
                            # block, where my own shardview of this view, extended past its box, addresses it
                            post_wait.append(copy_part(i, pb, bc, buf, unpack=True))
                            parts[i].append(_Source(pb, vcode[i], shard=shards[i], sv=vdist[i][w], received=True))
                            tape.ring_receives += 1
                        else:
                            parts[i].append(_Source(pb, vcode[i], buf=buf, cst=cst, received=True))
        if ops:
            # the pack kernels run on the current stream; NCCL orders its transfers after them.  The transfers are NOT
            # waited for here: ranges whose operands are all local (the interior of a stencil) are launched first and
            # overlap with them (the reference sends, then blocks in the receive loop, ramba/ramba.py:3646-3693)
            tape.p2p(ops)
    if shardview.is_empty(subspace):
        tape.wait()
        return tape.finish()
    # local parts
    for i in range(nviews):
        if i in gathered:
            continue
        sv = vdist[i][w]
        if local_everywhere[i] or shardview.is_compat(subspace, sv):
            parts[i].append(_Source(subspace, vcode[i], shard=shards[i], sv=sv))
        else:
            part = shardview.intersect(sv, exec_dist[w])
            if not shardview.is_empty(part):
                parts[i].append(_Source(shardview.clean_range(part), vcode[i], shard=shards[i],
                                        sv=sv if ring[i] else shardview.mapslice_keep(sv, part.start, part.start + part.size)))
    # ranges: every operand has one source inside a range
    single = builtins.all(len(p) == 1 and not p[0].received and (p[0].box is subspace or shardview.is_compat(p[0].box, subspace)) for p in parts)
    if single:
        ranges = [subspace]
    else:
        ranges = shardview.get_range_splits_list([shardview.clean_range(subspace)] + [s.box for p in parts for s in p])
        ranges = [r for r in ranges if not shardview.is_empty(r) and shardview.contains(subspace, r)]
    k = len(subspace.size)
    red_axes = list(red_axes) if red_axes else []
    order = red_axes + [d for d in range(k) if d not in red_axes]
    gred_out = None
    if gred:
        gred_out = [None] * len(prog.reds)
        for (slot, red_view) in gred:
            i = _view_index(views, red_view)
            # this worker's element of the partial array: the first element of its (size-1) block
            off, _ = RT.bind_view(vdist[i][w], shards[i].strides, shardview.clean_range(vdist[i][w]))
            gred_out[slot] = (shards[i].ptr(off), vcode[i])
    if ared:
        ared = [(slot, _view_index(views, red_view), REDUCTIONS[op].combine) for (slot, red_view, op) in ared]

    def source(i, r):
        for s in parts[i]:
            if shardview.contains(s.box, r):
                return s
        return None

    def needs_transfer(r):
        return builtins.any(s is not None and s.received for s in (source(i, r) for i in range(nviews)))

    def wait_and_unpack():
        tape.wait()
        for args in post_wait:
            tape.launch(*args)
        post_wait.clear()

    if tape.in_flight:
        ranges = sorted(ranges, key=lambda r: 1 if needs_transfer(r) else 0)  # (stable: local ranges first)
    for r in ranges:
        if tape.in_flight and needs_transfer(r):
            wait_and_unpack()
        bound = []
        for i in range(nviews):
            src = source(i, r)
            if src is None:
                raise ProgramError("internal: an operand has no source for range %r" % (r,))
            bound.append(src.bind(r))
        shape_r = [int(x) for x in r.size]
        gs = [int(x) for x in r.start]
        if ared:
            _axis_reduction(tape, prog, ared, order, len(red_axes), shape_r, gs, bound, w, W)
        else:
            tape.launch(prog, shape_r, gs, bound, reds=gred_out, worker_num=w, num_workers=W)
    wait_and_unpack()  # (nothing needed them, e.g. an empty boundary)
    return tape.finish()


def _axis_reduction(tape, prog, ared, order, nred, shape_r, gs, bound, w, W):
    """Axis reduction over one range: stage 1 (iteration dims permuted to `order`, the nred reduced dims first) into
    per-split partials, then per (slot, view index of its partial array, combine operator) in ared the fold of the splits
    and the combine."""
    shape_p = [shape_r[d] for d in order]
    gs_p = [gs[d] for d in order]
    bound_p = [(b[0], [b[1][d] for d in order], b[2]) + tuple(b[3:]) for b in bound]
    kept_elems = 1
    for d in range(nred, len(order)):
        kept_elems *= shape_p[d]
    red_len = 1
    for d in range(nred):
        red_len *= shape_p[d]
    kept_work = max(1, kept_elems // 4)
    target = 132 * 2048  # H100 SXM: 132 SMs x 2048 resident threads
    nsplit = 1 if kept_work >= target else builtins.min(builtins.max(1, red_len // 8), -(-target // kept_work))
    partials = tape.empty(len(prog.reds) * nsplit * kept_elems + 1, torch.float64)
    tape.launch(_remap_iota(prog, order), shape_p, gs_p, bound_p, n_axis_red=nred, axis_nsplit=nsplit,
                axis_partials=partials.data_ptr(), worker_num=w, num_workers=W)
    kept_shape = shape_p[nred:]
    cst, _ = _contig_strides(kept_shape)
    for (slot, i, combine) in ared:
        rop, rct = prog.reds[slot]
        acc_code = cabi.F64 if rct == cabi.T_F64 else cabi.I64
        tot_ptr = partials.data_ptr() + slot * nsplit * kept_elems * 8
        if nsplit > 1:
            tot = tape.empty(kept_elems + 1, torch.float64)
            tape.reduce_partials(tot.data_ptr(), tot_ptr, kept_elems, nsplit, kept_elems, acc_code, rop)
            tot_ptr = tot.data_ptr()
        rb = bound_p[i]
        tape.launch(_combine_program(rb[2], acc_code, combine), kept_shape, gs_p[nred:],
                    [(rb[0], rb[1][nred:], rb[2]), (tot_ptr, cst, acc_code)])


def _remap_iota(prog, order):
    """Iteration dims were permuted to `order`: point IOTA operands at the new positions."""
    if not prog.uses_iota:
        return prog
    memo = prog.__dict__.setdefault("_remapped", {})
    hit = memo.get(tuple(order))
    if hit is not None:
        return hit  # (one object per permutation: it keys the launch memo)
    p = copy.copy(prog)
    p.__dict__.pop("_remapped", None)
    p.__dict__.pop("_packed", None)
    inv = {d: i for i, d in enumerate(order)}
    p.insns = []
    for f in prog.insns:
        g = dict(f)
        for nm in ("a", "b", "c"):
            if g[nm + "_kind"] == cabi.K_IOTA:
                g[nm + "_idx"] = inv[g[nm + "_idx"]]
        p.insns.append(g)
    p.uses_iota = {inv[d] for d in prog.uses_iota}
    memo[tuple(order)] = p
    return p
