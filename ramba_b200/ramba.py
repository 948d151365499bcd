"""ramba_b200.ramba — array handles, operator tables and the deferred-op fuser.

Drop-in for the part of `ramba.ramba` that lies on the fused elementwise / reduction /
shifted-slice path (SURVEY.md §8a):

  bdarray / ndarray        ramba/ramba.py:1049-1158, 5409-6901
  op tables + make_method  ramba/ramba.py:7842-7993
  deferred_op              ramba/ramba.py:8039-8533  (do_ops / execute keep their call shape; add_op takes one
                           Statement record instead of the alternating "code string, operand" oplist)
  creation / sync          ramba/ramba.py:8563-8991, 9843-9849

Each API call writes one Statement (`dst = expr`, or a reduction by op name over its axes) through DAG.assign /
DAG.reduce; the DAG hands it to the current fused op; nothing runs until a flush (sync(),
asarray(), a scalar read, or an incompatible op).  At flush, arrays whose Python handle is dead
never touch HBM (they are register temporaries), live ones are read/written in place
(ramba/ramba.py:8123-8127).  Execution is SPMD: every rank runs this driver code and executes its
own division on its own GPU through ramba_b200.runtime.
"""
import builtins
import os
import numbers
import weakref

import numpy as np
import torch

from . import _cabi as cabi
from . import advindex
from . import argreduce
from . import binning
from . import quantile as _quantile_mod
from . import compaction
from . import blocks
from . import common
from . import shardview
from .common import dprint, timer, add_time
from .flush import _contig_strides, _pack_program, _plan_cache, run_deferred_ops
from .program import E, REDUCTIONS, Iota, Lowering, ProgramError, ProgramLimit, dtype_class, fold_expr, getminmax, rb_dtype, red_identity
from .runtime import RT, torch_dtype

int64 = np.int64
float64 = np.float64
float32 = np.float32

_gid_counter = [0]


def _new_gid():
    """Deterministic ids so that all SPMD ranks agree (ramba/ramba_uuid.py:15-31)."""
    _gid_counter[0] += 1
    return _gid_counter[0]


def shapeToInt(shape):
    if type(shape) is tuple:
        for x in shape:
            if type(x) is not int:
                break
        else:
            return shape
    if isinstance(shape, numbers.Integral):
        return (int(shape),)
    return tuple(int(x) if isinstance(x, numbers.Integral) else x for x in shape)


# =============================================================================================
# bdarray: the physical distributed buffer
# =============================================================================================
class bdarray:
    """remote_constructed: the array's blocks exist (a flush or blocks.block made them).  flex_dist: its partition can
    still be pinned to that of the fused op it is used in.  Whatever sets remote_constructed clears flex_dist, so
    flex_dist implies not remote_constructed."""

    __slots__ = ("shape", "gid", "pad", "distribution", "nrefs", "remote_constructed", "flex_dist", "dtype", "failed")

    def __init__(self, shape, distribution, gid, pad, fdist, dtype):
        self.shape = shape
        self.gid = gid
        self.pad = pad
        self.distribution = distribution
        self.nrefs = 0
        self.remote_constructed = False
        self.flex_dist = fdist
        self.dtype = np.dtype(dtype)
        self.failed = None  # why the last fused op that wrote this array did not run (its contents are undefined then)

    def ndarray_del_callback(self):
        self.nrefs -= 1
        if self.nrefs < 1:
            deferred_op.del_remote_array(self.gid)

    @classmethod
    def assign_bdarray(cls, nd, shape, base=None, distribution=None, pad=0, flexible_dist=False, dtype=None, **kwargs):
        """The buffer of a new handle: `base`'s (a bdarray) for a view, else a new one."""
        bd = base
        if bd is None:
            if dtype is None:
                dtype = np.float64
            if shape == ():
                distribution = np.zeros((), dtype=dtype)
            elif distribution is None:
                distribution = shardview.default_distribution(shape, **kwargs) if kwargs else shardview.default_distribution_of(shape)
            else:
                # a new array: same boxes, fresh buffer coordinates
                distribution = shardview.clean_dist(distribution)
            bd = cls(shape, distribution, _new_gid(), pad, flexible_dist, dtype)
        bd.nrefs += 1
        return bd


class ndarray_details:
    __slots__ = ("shape", "distribution", "dtype", "local_border")

    def __init__(self, nd):
        self.shape = nd.shape
        self.distribution = nd.distribution
        self.dtype = nd.dtype
        self.local_border = nd.local_border


# =============================================================================================
# the fuser
# =============================================================================================
class ArrRef:
    """What a statement remembers about an array operand.  Statements must not keep the Python
    handle alive: whether a temporary is materialised depends on its handle being dead at flush
    time (ramba/ramba.py:8123-8127; the reference keeps only variable names + the bdarray)."""

    __slots__ = ("gid", "distribution", "shape", "dtype", "local_border", "bd")

    def __init__(self, nd):
        self.gid = nd.gid
        self.distribution = nd.distribution
        self.shape = nd.shape
        self.dtype = nd.dtype
        self.local_border = nd.local_border
        self.bd = nd.bdarray


def _raise_failed(bd):
    raise RuntimeError("this array was to be written by a fused op that failed (%s): its contents are undefined" % (bd.failed,))


def _ref_of(nd):
    """The ArrRef of a handle (one per handle: a handle's shape, partition and buffer never change)."""
    r = nd._ref
    if r is None:
        r = nd._ref = ArrRef(nd)
    return r


def _detach(x, reads, direct):
    """The expression with every array leaf replaced by its ArrRef (the handle appended to `reads`, in order of appearance)
    and every 0-d array leaf by the value it holds NOW (0-d arrays keep their value on the host and can be assigned to
    before a deferred statement runs).  That value is a NumPy scalar in a statement the DAG defers and a Python scalar in
    one that goes `direct`ly to the fuser: the lowering types a scalar by its type."""
    if isinstance(x, E):
        return E(x.op, *[_detach(a, reads, direct) for a in x.args], imm=x.imm)
    if isinstance(x, ndarray):
        if x.shape == ():
            return x.distribution.item() if direct else x.distribution[()]
        reads.append(x)
        return _ref_of(x)
    return x


class Statement:
    """One deferred statement, as the API call wrote it.  An assignment (op None) is `dst = expr` at every index of dst,
    where dst's mask (its maskarray) is true; a reduction is `dst = dst (op) expr` reduced over `axes` (None: every axis),
    dst being the partial array's view broadcast to the source's shape.  expr is an E tree over ArrRefs, scalars and Iota;
    `reads` holds the handles of its array operands, which keep them alive while the statement waits in the DAG.
    deferred_op.add_op replaces dst and mask by their ArrRefs and drops `reads`: a pending fused op holds no handle."""

    __slots__ = ("dst", "expr", "reads", "mask", "op", "axes", "elide")

    def __init__(self, dst, expr, reads, op=None, axes=None, elide=None):
        self.dst, self.expr, self.reads, self.mask = dst, expr, reads, dst.maskarray
        self.op, self.axes, self.elide = op, axes, elide


def _other_view(dists, dist):
    """True when one of `dists` (None: a partition that was still flexible) is not `dist`."""
    for d in dists:
        if d is not None and not shardview.dist_is_eq(d, dist):
            return True
    return False


def _walk_operands(x, out):
    if isinstance(x, E):
        for a in x.args:
            _walk_operands(a, out)
    else:
        out.append(x)
    return out


_lower_cache = {}
_VERIFY_LOWER_CACHE = bool(int(os.environ.get("RB200_VERIFY_LOWER_CACHE", "0")))


def _check_same_lowering(a, b):
    """RB200_VERIFY_LOWER_CACHE=1: every memoised lowering is recomputed and must be identical."""
    if a[0] != b[0]:
        raise AssertionError("lowering memo: %r vs %r" % (a[0], b[0]))
    if a[0] == "limit":
        return
    pa, pb = a[1], b[1]
    same = (pa.insns == pb.insns and pa.scalars == pb.scalars and pa.n_regs == pb.n_regs and pa.reds == pb.reds
            and pa.view_written == pb.view_written and pa.uses_iota == pb.uses_iota and a[2] == b[2] and a[3] == b[3])
    if not same:
        raise AssertionError("lowering memo returned a different op list for the same structural key")


class _Use:
    """What the pending fused op knows about one array its statements touch.
      bd        the array's bdarray, held until the flush pins its partition and marks its blocks made
      reads     the distributions statements read the array through (None where its partition was still flexible)
      writes    the same for the statements that store into it
      flexible  its partition was flexible at its first admission: the flush pins it to the op's
      resident  its blocks existed at an admission: the flush keeps it in memory even if every handle has died"""

    __slots__ = ("bd", "reads", "writes", "flexible", "resident")

    def __init__(self, bd):
        self.bd = bd
        self.reads = []
        self.writes = []
        self.flexible = bd.flex_dist
        self.resident = False


class deferred_op:
    ramba_deferred_ops = None
    max_statements = 40

    def __init__(self, shape, distribution, fdist):
        self.shape = shape
        self.distribution = distribution
        self.flex_dist = fdist
        self.arrays = {}    # gid -> _Use, for every array a statement of this op reads, stores or reduces into
        self.dead = set()   # arrays whose last handle died while this op was pending
        self.elide = set()  # arrays proven unobservable after the flush (dying temporaries of a reduction)
        self.statements = []
        self.red_axes = None  # the axes every axis reduction of this op reduces over (ramba/ramba.py:8425-8432)

    def _use(self, nd):
        """The record of nd's array, made at its first admission; marks it resident when its blocks exist now."""
        bd = nd.bdarray
        u = self.arrays.get(bd.gid)
        if u is None:
            u = self.arrays[bd.gid] = _Use(bd)
        if bd.remote_constructed:
            u.resident = True
        return u

    # ---- adding statements --------------------------------------------------------------
    @classmethod
    def add_op(cls, stmt):
        """Admit Statement `stmt` to the pending fused op, flushing that first if the two cannot fuse (the operator seam,
        ramba/ramba.py:8383-8385).  A reduction's `elide` names the gid of an operand that nobody can observe once the
        calling API function returns (the temporary of `(X*2.0 + 1.0).sum()`): it is treated as dead in the flush that
        holds this statement, provided the statement that writes it is part of the SAME fused op."""
        t0 = timer()
        dst, reads = stmt.dst, stmt.reads
        # (a global reduction only accumulates into its partial view, through a reduction slot: it neither reads nor
        # stores that view element by element)
        stores = stmt.op is None or stmt.axes is not None
        operands = [dst] + reads if stores and dst.shape != () else reads
        shape, distribution = dst.shape, dst.distribution
        abd = dst.bdarray
        # the partition of `dst` can still follow the op's only if dst is a whole array that no flush has touched: a VIEW of
        # a flexible array was cut from the partition the array had then and does not move when the array is pinned
        fixed = not abd.flex_dist or dst.base is not None
        cur = cls.ramba_deferred_ops
        if cur is not None:
            if (cur.shape != shape
                    or (fixed and not cur.flex_dist and not shardview.compatible_distributions(cur.distribution, distribution))
                    or len(cur.statements) >= cls.max_statements):
                cls.do_ops()
                cur = None
            elif cur.red_axes is not None and stmt.axes != cur.red_axes:
                # reductions on an axis must agree (ramba/ramba.py:8425-8432); a plain statement after an axis reduction
                # would run once per reduced element
                cls.do_ops()
                cur = None
        # alias check 1: reads/writes a shifted version of an array written earlier in this op
        if cur is not None:
            for o in operands:
                u = cur.arrays.get(o.gid)
                if u is not None and _other_view(u.writes, o.distribution):
                    cls.do_ops()
                    cur = None
                    break
        # alias check 2: writes an array that is also read through a different view
        if stores:
            hit = False
            for o in operands:
                if o is not dst and o.gid == abd.gid and not shardview.dist_is_eq(o.distribution, distribution):
                    hit = True
                    break
            if not hit and cur is not None:
                u = cur.arrays.get(abd.gid)
                hit = u is not None and _other_view(u.reads, distribution)
            if hit:
                tmp_array = empty_like(dst)
                cls.add_op(Statement(tmp_array, stmt.expr, reads))
                cls.do_ops()
                cls.add_op(Statement(dst, _ref_of(tmp_array), [tmp_array]))
                return
        if cur is None:
            cur = cls.ramba_deferred_ops = cls(shape, distribution, not fixed)
        if fixed and (cur.flex_dist or not abd.flex_dist):
            cur.distribution = distribution
            cur.flex_dist = False
        u = cur.arrays.get(stmt.elide) if stmt.elide is not None else None
        if u is not None and u.writes and not u.bd.remote_constructed:
            # (decided HERE, after admission: a flush forced by this very statement must still materialise the operand)
            cur.elide.add(stmt.elide)
        mask = stmt.mask
        if stores:
            if mask is not None:
                operands = [mask] + operands
            if dst.shape != ():  # (like the operand list above, the op keeps no record of a 0-d destination)
                cur._use(dst).writes.append(None if abd.flex_dist else distribution)
        for x in operands:
            xbd = x.bdarray
            if xbd.failed is not None:
                _raise_failed(xbd)
            cur._use(x).reads.append(None if xbd.flex_dist else x.distribution)
        if stmt.op is not None:
            cur._use(dst)
            if stmt.axes is not None:
                cur.red_axes = stmt.axes
        stmt.dst = _ref_of(dst)
        stmt.mask = _ref_of(mask) if mask is not None else None
        stmt.reads = None
        cur.statements.append(stmt)
        add_time("deferred_ops::add_op", timer() - t0)

    @classmethod
    def del_remote_array(cls, gid):
        if cls.ramba_deferred_ops is None:
            RT.destroy_array(gid)
        else:
            cls.ramba_deferred_ops.dead.add(gid)

    @classmethod
    def do_ops(cls):
        if cls.ramba_deferred_ops is not None:
            cur = cls.ramba_deferred_ops
            cls.ramba_deferred_ops = None
            cur.execute()

    # ---- flush ---------------------------------------------------------------------------
    def execute(self):
        """Run the op.  An array lives in memory if its blocks existed at an admission or someone can still read it after
        the flush; every other array is a register temporary."""
        t0 = timer()
        dead, elide = self.dead, self.elide
        live = {g for (g, u) in self.arrays.items() if u.resident or (g not in dead and g not in elide)}
        self._pin(live)
        try:
            self._run_statements(self.statements, live)
        except BaseException as ex:
            # the statements of this op are gone: what they were to write is undefined from here on.  Reading it later must
            # fail loudly, not return whatever the shard holds (the reference re-raises on the driver and stops there,
            # ramba/ramba.py:3875-3881, 4053-4054)
            why = "%s: %s" % (type(ex).__name__, str(ex)[:300])
            for u in self.arrays.values():
                if u.writes:
                    u.bd.failed = why
            raise
        finally:
            self._finish(live)
        add_time("driver_deferred_op", timer() - t0)

    def _pin(self, gids):
        """Pin flexible distributions to the op's distribution (ramba/ramba.py:8130-8136)."""
        for g in gids:
            u = self.arrays[g]
            if u.flexible and u.bd.shape == self.shape:
                u.bd.distribution[:] = shardview.clean_dist(self.distribution)

    def _run_statements(self, statements, live):
        """Lower `statements` to one op list and launch it.  The reference never fails on the length of a fused chain
        (Numba compiles whatever the fuser accumulated); a prebuilt library has table sizes (views, spill registers,
        instructions, scalars, reduction slots), so a chain that exceeds one of them is cut in two at a statement
        boundary and run as two launches: arrays that are written before the cut and read after it, and would
        otherwise have stayed register temporaries, are materialised for the duration of the flush."""
        try:
            lowered = self._lower(statements, live)
        except ProgramLimit:
            if len(statements) < 2:
                raise
            m = len(statements) // 2
            first, second = statements[:m], statements[m:]
            written = {st.dst.gid for st in first if st.op is None}
            crossing = set()
            for st in second:
                for x in (st.expr, st.mask):
                    for o in _walk_operands(x, []):
                        if isinstance(o, ArrRef) and o.gid in written and o.gid not in live:
                            crossing.add(o.gid)
            self._pin(crossing)
            both = live | crossing
            try:
                self._run_statements(first, both)
                self._run_statements(second, both)
            finally:
                for g in crossing:
                    RT.destroy_array(g)
            return
        if lowered is None:
            return
        views, prog, gred, ared = lowered
        if common.debug_showcode and common.worker_num == 0:
            print(format_program(prog, views, self.shape))
        t1 = timer()
        run_deferred_ops(views, prog, self.distribution, gred, ared, self.red_axes if ared else None)
        add_time("run_deferred_ops", timer() - t1)

    def _lower(self, statements, live):
        """Statements -> (view table, op list, global reductions, axis reductions).  The op list depends only on the
        STRUCTURE of the statements (operators, which operand is which view / temporary / dead array, view dtypes and
        aliasing, scalar values), not on the arrays themselves, so it is memoised on that structure: the second and
        later iterations of a loop skip typing, lowering and register allocation (the reference gets the same effect
        from Numba's compile cache keyed by the generated source, ramba/ramba.py:8247-8265)."""
        views = []  # (gid, details)
        vindex = {}
        reads = {}
        gid_ids = {}
        elide = self.elide

        def view_of(nd):
            lst = vindex.setdefault(nd.gid, [])
            for (dist, idx) in lst:
                if dist is nd.distribution or shardview.dist_is_eq(dist, nd.distribution):
                    return idx
            idx = len(views)
            views.append((nd.gid, nd))
            lst.append((nd.distribution, idx))
            return idx

        def key_of(x):
            """Structural key of an expression; registers views in first-use order and counts their reads."""
            if isinstance(x, E):
                return (x.op, x.imm) + tuple([key_of(a) for a in x.args])
            if isinstance(x, ArrRef):
                if x.gid in live:
                    i = view_of(x)
                    reads[i] = reads.get(i, 0) + 1
                    return ("v", i)
                return ("d", gid_ids.setdefault(x.gid, len(gid_ids)))
            if isinstance(x, Iota):
                return ("i", x.dim)
            if isinstance(x, np.ndarray) and x.shape == ():
                x = x.item()
            return ("s", type(x), repr(x))

        skeys = []
        for st in statements:
            ek = key_of(st.expr)
            dst = st.dst
            if st.op is not None:
                skeys.append((st.op, st.axes is None, ek, view_of(dst)))
                continue
            mk = key_of(st.mask) if st.mask is not None else None
            if dst.gid in live:
                dk = ("v", view_of(dst))
            elif dst.gid in elide:
                dk = ("e", gid_ids.setdefault(dst.gid, len(gid_ids)), rb_dtype(dst.dtype))
            else:
                dk = ("d", gid_ids.setdefault(dst.gid, len(gid_ids)))
            skeys.append((None, dk, ek, mk))
        if len(views) > cabi.MAX_VIEWS:
            raise ProgramLimit("fused op touches %d array views (max %d)" % (len(views), cabi.MAX_VIEWS))
        if not views or not statements:
            return None
        vcodes = tuple([rb_dtype(det.dtype) for (_, det) in views])
        alias = {}
        key = (vcodes, tuple([alias.setdefault(g, len(alias)) for (g, _) in views]), tuple(skeys))
        hit = _lower_cache.get(key)
        if hit is None or _VERIFY_LOWER_CACHE:
            try:
                fresh = self._lower_uncached(statements, live, views, vindex, reads)
            except ProgramLimit as e:
                fresh = ("limit", str(e))
            if hit is not None:
                _check_same_lowering(hit, fresh)  # (verification mode; the memoised object stays, it keys the plan memo)
            else:
                if len(_lower_cache) >= 1024:
                    _lower_cache.clear()
                hit = _lower_cache[key] = fresh
        if hit[0] == "limit":
            raise ProgramLimit(hit[1])
        _, prog, gslots, aslots = hit
        gred = [(slot, statements[si].dst) for (slot, si) in gslots]
        ared = [(slot, statements[si].dst, statements[si].op) for (slot, si) in aslots]
        return views, prog, gred, ared

    def _lower_uncached(self, statements, live, views, vindex, reads):
        def view_of(nd):
            for (dist, idx) in vindex[nd.gid]:
                if dist is nd.distribution or shardview.dist_is_eq(dist, nd.distribution):
                    return idx
            raise ProgramError("internal: view not registered")

        lw = Lowering([rb_dtype(det.dtype) for (_, det) in views])
        lw.view_gids = [g for (g, _) in views]
        lw.note_view_reads(reads)
        dead_values = {}

        def resolve(o):
            if isinstance(o, ArrRef):
                if o.gid in live:
                    return lw.read_view(view_of(o))
                if o.gid in dead_values:
                    return dead_values[o.gid]
                return lw.scalar(0)  # read of an uninitialised, already dead array
            if isinstance(o, np.ndarray) and o.shape == ():
                return lw.scalar(o.item())
            return lw.scalar(o)

        gslots = []  # (slot, statement index)
        aslots = []
        for si, st in enumerate(statements):
            tv = lw.build(st.expr, resolve)
            if st.op is not None:
                (gslots if st.axes is None else aslots).append((lw.reduce(REDUCTIONS[st.op].code, tv), si))
                continue
            dst, mask = st.dst, st.mask
            if dst.gid in live:
                m = resolve(mask) if mask is not None else None
                lw.store(view_of(dst), tv, m)
            elif dst.gid in self.elide:
                # an elided temporary keeps the value a store + reload would have given it (the reference
                # materialises it: ramba_b200 only skips the memory traffic, not the rounding)
                dead_values[dst.gid] = lw.astype(tv, rb_dtype(dst.dtype))
            else:
                if mask is not None and dst.gid in dead_values:
                    # a masked assignment to an array that lives in a register: elements where the mask is false keep
                    # the value the array had (`t = a + b; t[m] = 0.5; r = cos(t)` with t never stored)
                    old = dead_values[dst.gid]
                    tv = lw.build(E("where", mask, lw.coerce(tv, old.cls), old), resolve)
                dead_values[dst.gid] = tv
        return ("ok", lw.finish(), gslots, aslots)

    def _finish(self, live):
        """Free the blocks of the arrays that died while the op was pending; every other array the flush kept in memory
        now has its blocks, at a fixed partition."""
        for g in self.dead:
            RT.destroy_array(g)
        for g in live:
            if g not in self.dead:
                bd = self.arrays[g].bd
                bd.remote_constructed = True
                bd.flex_dist = False


# =============================================================================================
# the lazy DAG in front of the fuser (ramba/ramba.py:4387-5293)
# =============================================================================================
NO_DAG = bool(int(os.environ.get("RAMBA_NO_DAG", "0")))  # the reference's switch (ramba/common.py): statements go straight to the fuser


class DAG:
    """One node per deferred STATEMENT (`dst = expr`, a reduction, a fill).  The reference builds one node per API call
    and runs the call's executor when the node is materialised (DAG.add ramba/ramba.py:4512-4548, DAGapi 5160-5293);
    here an API call computes its result's shape / dtype / distribution at once (all metadata, nothing on the GPU) and
    what is deferred is exactly the part the reference's executors end in: the `deferred_op.add_op` of the statement.

      * dependencies are tracked per bdarray (gid): a node depends on the last pending writer of everything it reads
        (RAW), and a writer on the last pending writer (WAW) and on every pending reader since (WAR) - what the
        reference gets from `ndarray.dag` / `bdarray.dag` and the in-place rule of DAG.add (4527-4539);
      * `instantiate(arr)` walks the backward dependencies of arr's last writer depth first, same-shaped branches
        first (depth_first_traverse, 4792-4838), hands the statements to the fuser in that order and flushes;
        `execute_all` (sync) starts from every node nothing depends on, oldest first, grouped by shape (5080-5105) -
        so interleaved chains over different shapes fuse per shape instead of flushing at every change;
      * a node whose output nobody can observe is never executed (DAG.execute's `soutput is None`, 4846-4849): the
        destination of an out-of-place statement is held weakly; when the last handle dies the node is dropped together
        with the handles it holds, which may drop the nodes that produced those, and so on;
      * nodes hold their operands strongly until they are executed (like the reference's `args`), so whether a
        temporary is materialised is still decided by handle liveness at flush time;
      * while a node executes, API calls made by the executor run inline (`DAG.in_evaluate`), and RAMBA_NO_DAG=1
        makes every call inline."""

    __slots__ = ("seq_no", "stmt", "out_ref", "shape", "backward_deps", "forward_deps", "executed", "rgids", "wgid",
                 "__weakref__")
    pending = {}       # seq_no -> node, in program order
    last_writer = {}   # gid -> pending node that writes the array last
    readers = {}       # gid -> pending nodes that read it since
    in_evaluate = 0
    dag_count = 0
    executed_count = 0
    pruned_count = 0
    max_pending = 4096

    @classmethod
    def assign(cls, dst, expr):
        """Defer `dst = expr` (where dst's mask is true)."""
        cls._add(dst, expr, None, None, None)

    @classmethod
    def reduce(cls, op, expr, red_view, axes=None, elide=None):
        """Defer reduction `op` (sum prod min max all any) of expr over `axes` (None: every axis) into the partial array
        view red_view; `elide`: see deferred_op.add_op."""
        cls._add(red_view, expr, op, axes, elide)

    @classmethod
    def _add(cls, dst, expr, op, axes, elide):
        direct = NO_DAG or cls.in_evaluate
        reads = []
        stmt = Statement(dst, _detach(expr, reads, direct), reads, op, axes, elide)
        if direct:
            deferred_op.add_op(stmt)
            return
        node = object.__new__(cls)
        seq = node.seq_no = cls.dag_count
        cls.dag_count = seq + 1
        node.stmt = stmt
        node.executed = False
        node.forward_deps = set()
        node.shape = dst.shape
        rg = [o.bdarray.gid for o in reads]
        if stmt.mask is not None:
            rg.append(stmt.mask.gid)
        wgid = dst.bdarray.gid
        # the destination of an out-of-place statement is the only way to observe it: hold it weakly
        if op is None and dst.base is None and stmt.mask is None and wgid not in rg:
            stmt.dst = None
            node.out_ref = weakref.ref(dst, node._output_died)
        else:
            node.out_ref = None
        lw, rd = cls.last_writer, cls.readers
        deps = []
        if lw:
            for g in rg + [wgid]:
                d = lw.get(g)
                if d is not None and d not in deps:
                    deps.append(d)
        if rd:
            for d in rd.pop(wgid, ()):
                if d not in deps:
                    deps.append(d)
        for d in deps:
            d.forward_deps.add(node)
        node.backward_deps = deps
        node.rgids = rg
        node.wgid = wgid
        for g in rg:
            lst = rd.get(g)
            if lst is None:
                rd[g] = [node]
            else:
                lst.append(node)
        lw[wgid] = node
        cls.pending[node.seq_no] = node
        if len(cls.pending) >= cls.max_pending:
            cls.execute_all()

    # ---- pruning ---------------------------------------------------------------------------
    def _output_died(self, _ref=None):
        """Weakref callback: the last handle of this node's (out-of-place) destination is gone."""
        try:
            if self.executed or DAG.in_evaluate:
                return  # (during an evaluation the execution loop skips it)
            if not self.forward_deps:
                self._retire(False)
        except Exception:  # (interpreter shutdown: module globals may be gone)
            pass

    def _retire(self, ran):
        """Take the node out of the graph (executed or pruned) and let go of its operands."""
        self.executed = True
        cls = DAG
        cls.pending.pop(self.seq_no, None)
        for d in self.backward_deps:
            d.forward_deps.discard(self)
        for f in self.forward_deps:
            try:
                f.backward_deps.remove(self)
            except ValueError:
                pass
        lw, rd = cls.last_writer, cls.readers
        if lw.get(self.wgid) is self:
            del lw[self.wgid]
        for g in self.rgids:
            lst = rd.get(g)
            if lst is not None:
                try:
                    lst.remove(self)
                except ValueError:
                    pass
                if not lst:
                    del rd[g]
        if ran:
            cls.executed_count += 1
        else:
            cls.pruned_count += 1
        self.backward_deps = ()
        self.forward_deps = ()
        self.out_ref = None
        # last: dropping the operands may end other arrays' lives (and prune their producers through the callback above)
        self.stmt = None

    def _execute(self):
        """Hand the statement to the fuser (DAG.execute, ramba/ramba.py:4846-4872)."""
        stmt = self.stmt
        if self.out_ref is not None:
            stmt.dst = self.out_ref()
            if stmt.dst is None:
                self._retire(False)  # nobody can observe the result
                return
        self._retire(True)
        deferred_op.add_op(stmt)

    # ---- materialisation -------------------------------------------------------------------
    @classmethod
    def _run(cls, roots):
        """Depth-first over the backward dependencies of `roots` (same-shaped branches first), then execute in that
        order (depth_first_traverse + the loop of instantiate_dag_node, ramba/ramba.py:4792-4838, 5007-5012)."""
        order = []
        seen = set()
        for root in roots:
            if root.executed or root in seen:
                continue
            seen.add(root)
            stack = [(root, iter(cls._ordered_deps(root)))]
            while stack:
                n, it = stack[-1]
                for d in it:
                    if d not in seen and not d.executed:
                        seen.add(d)
                        stack.append((d, iter(cls._ordered_deps(d))))
                        break
                else:
                    order.append(n)
                    stack.pop()
        cls.in_evaluate += 1
        try:
            for n in order:
                if not n.executed:
                    n._execute()
        finally:
            cls.in_evaluate -= 1

    @staticmethod
    def _ordered_deps(node):
        deps = node.backward_deps
        if len(deps) < 2:
            return deps
        shp = node.shape
        return [d for d in deps if d.shape == shp] + [d for d in deps if d.shape != shp]

    @classmethod
    def instantiate(cls, arr=None):
        """Make `arr` real: run what it depends on, then flush (DAG.instantiate, ramba/ramba.py:4833-4844)."""
        if cls.pending and isinstance(arr, ndarray):
            node = cls.last_writer.get(arr.gid)
            if node is not None:
                cls._run([node])
        deferred_op.do_ops()

    @classmethod
    def before_write(cls, arr):
        """Make arr's storage safe to overwrite outside a fused op: run every pending statement that reads it (WAR) and
        the last one that writes it (WAW), then flush."""
        g = arr.gid
        nodes = list(cls.readers.get(g, ()))
        if g in cls.last_writer:
            nodes.append(cls.last_writer[g])
        if nodes:
            cls._run(nodes)
        deferred_op.do_ops()

    @classmethod
    def execute_all(cls, do_ops=False):
        """Run every pending node: start from the ones nothing depends on, oldest first, grouped by output shape
        (DAG.execute_all, ramba/ramba.py:5080-5105)."""
        if cls.pending:
            by_shape = {}
            for n in cls.pending.values():
                if not n.forward_deps:
                    by_shape.setdefault(n.shape, []).append(n)
            cls._run([n for lst in by_shape.values() for n in lst])
            if cls.pending:  # (nodes retired by the run may have left others without dependants)
                cls._run(list(cls.pending.values()))
        if do_ops:
            deferred_op.do_ops()

    @classmethod
    def reset(cls):
        """Forget every pending node without executing it (tests)."""
        for n in list(cls.pending.values()):
            n._retire(False)
        cls.pending.clear()
        cls.last_writer.clear()
        cls.readers.clear()
        cls.in_evaluate = 0
        deferred_op.ramba_deferred_ops = None


RT.on_reset.append(DAG.reset)


def format_program(prog, views, shape):
    """RAMBA_SHOW_CODE: print the op list (the reference prints the generated Python,
    ramba/ramba.py:8266-8284)."""
    kinds = ["-", "acc", "r", "v", "s", "iota"]
    cls = ["f64", "f32", "i64"]
    lines = ["fused op over %s: %d insns, %d regs, %d views" % (shape, len(prog.insns), prog.n_regs, len(views))]
    for i, f in enumerate(prog.insns):
        def opnd(p):
            k = f[p + "_kind"]
            if k == 0:
                return ""
            return kinds[k] + (str(f[p + "_idx"]) if k != 1 else "")
        extra = ""
        if f["st_reg"] != cabi.NOSTORE:
            extra += " ->r%d" % f["st_reg"]
        if f["st_view"] != cabi.NOSTORE:
            extra += " ->v%d" % f["st_view"]
        lines.append("  %2d: %-8s %s %s %s %s%s" % (i, cabi.OPS[f["op"]], cls[f["ctype"]], opnd("a"), opnd("b"), opnd("c"), extra))
    for i, (gid, det) in enumerate(views):
        lines.append("  v%d: gid %s %s %s" % (i, gid, det.shape, det.dtype))
    return "\n".join(lines)


# =============================================================================================
# ndarray
# =============================================================================================
def unify_args(lhs, rhs, dtype):
    """Result dtype of a binary op (ramba/ramba.py:4170-4191)."""
    rhs_dtype = rhs.dtype if hasattr(rhs, "dtype") else None
    if dtype is not None:
        if dtype == "float":
            if rhs_dtype is None:
                try:
                    rhs_dtype = np.dtype(type(rhs))
                except Exception:
                    rhs_dtype = None
            dtype = np.float32 if (rhs_dtype == np.float32 and lhs == np.float32) else np.float64
        return np.dtype(dtype)
    try:
        return np.result_type(lhs, rhs)
    except Exception:
        return np.result_type(lhs, rhs_dtype)


def numpy_broadcast_shape(a, b):
    def shp(x):
        if isinstance(x, tuple):
            return x
        if isinstance(x, (ndarray, np.ndarray)):
            return x.shape
        if isinstance(x, numbers.Number):
            return ()
        return (1,)

    sa, sb = shp(a), shp(b)
    if (isinstance(a, numbers.Number) or sa == ()) and (isinstance(b, numbers.Number) or sb == ()):
        return None
    if sa == sb or sb == ():  # (the common cases: same shape, array with scalar)
        return sa
    if sa == ():
        return sb
    return tuple(np.broadcast_shapes(sa, sb))


def canonical_dim(dim, dim_size, end=False, neg_slice=False, checkbounds=False, axis=0):
    if not isinstance(dim, (numbers.Integral, type(None))):
        raise TypeError("indices must be integer or None")
    if dim is None:
        dim = dim_size if end != neg_slice else 0
        dim -= 1 if neg_slice else 0
        return dim
    if dim < -dim_size:
        if checkbounds:
            raise IndexError(f"index {dim} out of bounds for axis {axis} with size {dim_size}")
        return -1 if neg_slice else 0
    elif dim < 0:
        return dim + dim_size
    elif dim < dim_size:
        return dim
    else:
        if checkbounds:
            raise IndexError(f"index {dim} out of bounds for axis {axis} with size {dim_size}")
        return dim_size - 1 if neg_slice else dim_size


def canonical_slice(sl, dim_size):
    s = 1 if sl.step is None else sl.step
    if not isinstance(s, numbers.Integral):
        raise TypeError("step must be integer or None")
    if s == 0:
        raise TypeError("step cannot be zero")
    return slice(canonical_dim(sl.start, dim_size, neg_slice=(s < 0)),
                 canonical_dim(sl.stop, dim_size, end=True, neg_slice=(s < 0)), int(s))


def canonical_index(index, shape):
    if not isinstance(index, tuple):
        index = (index,)
    if len(index) > len(shape):
        raise IndexError(f"too many indices for array: array is {len(shape)}-dimensional, but {len(index)} were indexed")
    out = []
    for i in range(len(shape)):
        if i >= len(index):
            out.append(slice(0, shape[i], 1))
            continue
        ti = index[i]
        if isinstance(ti, numbers.Integral):
            ni = canonical_dim(ti, shape[i], checkbounds=True, axis=i)
            out.append(slice(ni, ni + 1, 1))
        elif isinstance(ti, slice):
            out.append(canonical_slice(ti, shape[i]))
        else:
            raise IndexError("unsupported index term %r on the fused path" % (ti,))
    return tuple(out)


def _slice_len(s):
    if s.step > 0:
        return builtins.max(0, -(-(s.stop - s.start) // s.step))
    return builtins.max(0, -(-(s.start - s.stop) // (-s.step)))


class ReshapeError(Exception):
    """A reshape that would have to move data between shards (ramba/ramba.py: ReshapeError)."""


class ndarray_flags:
    __slots__ = ("arr",)

    def __init__(self, arr):
        self.arr = arr

    def __getitem__(self, item):
        if not isinstance(item, str):
            assert len(item) == 1
            item = item[0]
        if item == "WRITEABLE":
            return self.writeable
        raise KeyError(item)

    @property
    def writeable(self):
        return not self.arr.readonly

    @writeable.setter
    def writeable(self, val):
        # read-only is checked when a statement is issued (in program order), so the flag changes at once; a view of a
        # read-only base cannot be made writeable (NumPy's rule)
        if val and self.arr.base is not None and self.arr.base.readonly:
            raise ValueError("cannot set WRITEABLE flag to True of this array")
        self.arr.readonly = not val


class ndarray:
    __slots__ = ("base", "bdarray", "shape", "distribution", "local_border", "readonly", "maskarray", "_slices", "_ref", "__weakref__")
    __array_priority__ = 20.0

    def __init__(self, shape, dtype=None, *, base=None, distribution=None, local_border=0, flex_dist=True,
                 readonly=False, maskarray=None, **kwargs):
        if isinstance(shape, ndarray):  # copy constructor
            o = shape
            base, distribution, local_border, dtype = o.base if o.base is not None else o, o.distribution, o.local_border, o.dtype
            flex_dist, readonly, maskarray, shape = o.bdarray.flex_dist, o.readonly, o.maskarray, o.shape
        self.base = base
        if base is not None and base.readonly:
            readonly = True
        shape = shapeToInt(shape)
        self.bdarray = bdarray.assign_bdarray(self, shape, base.bdarray if base is not None else None, distribution, local_border,
                                              flex_dist, dtype, **kwargs)
        self.shape = shape
        self.distribution = distribution if (distribution is not None and base is not None) else self.bdarray.distribution
        self.local_border = local_border
        self.readonly = readonly
        self.maskarray = maskarray
        self._slices = None  # index -> (shape, distribution) of slice views taken so far
        self._ref = None     # what statements remember about this handle (ArrRef), made on first use

    def __del__(self):
        try:
            self.bdarray.ndarray_del_callback()
        except Exception:
            pass

    # ---- properties
    @property
    def gid(self):
        return self.bdarray.gid

    @property
    def dtype(self):
        return self.bdarray.dtype

    @property
    def ndim(self):
        return len(self.shape)

    @property
    def size(self):
        return int(np.prod(self.shape)) if self.shape else 1

    def __len__(self):
        return self.shape[0]

    @property
    def T(self):
        return self.transpose()

    def get_details(self):
        return ndarray_details(self)

    def instantiate(self):
        DAG.instantiate(self)
        return self

    @property
    def flags(self):
        """`arr.flags.writeable` / `arr.flags["WRITEABLE"]` (ndarray_flags, ramba/ramba.py:5365-5385)."""
        return ndarray_flags(self)

    # ---- host round trip (ramba/ramba.py:5735-5765)
    def asarray(self, out=None, non_blocking=False):
        """NumPy copy of the whole array on every rank.  ramba_b200 extensions: `out`, a preallocated
        C-contiguous host array (e.g. a view of pinned memory) to fill; `non_blocking=True` (single
        rank, pinned `out`) only enqueues the device->host copy on the current CUDA stream — the
        caller synchronises before reading `out` (lets transfers of different streams overlap)."""
        if self.shape == ():
            return self.distribution
        DAG.instantiate(self)
        return gather_to_host(self, out=out, non_blocking=non_blocking)

    def __array__(self, dtype=None, copy=None):
        a = self.asarray()
        return a if dtype is None else a.astype(dtype)

    def item(self):
        a = self.asarray()
        return a.item()

    def __float__(self):
        return float(self.item())

    def __int__(self):
        return int(self.item())

    def __bool__(self):
        return bool(self.item())

    def __index__(self):
        return int(self.item())

    def __repr__(self):
        return "ramba_b200.ndarray(" + repr(self.asarray()) + ")"

    def copy(self):
        return copy(self)

    # ---- elementwise machinery (ramba/ramba.py:5768-5786, 6055-6139)
    @classmethod
    def broadcast(cls, a, b):
        new_shape = numpy_broadcast_shape(a, b)

        def view(x):
            if isinstance(x, ndarray) and x.shape == ():
                return x.distribution[()]  # (the VALUE, now: a 0-d array may be assigned to before the statement runs)
            if not isinstance(x, ndarray) or new_shape == x.shape:
                return x
            return x.broadcast_to(new_shape)

        return new_shape, view(a), view(b)

    def broadcast_to(self, shape):
        shape = shapeToInt(shape)
        new_dims = len(shape) - len(self.shape)
        if new_dims < 0 or builtins.any(a > 1 and b > 1 and a != b for a, b in zip(shape[new_dims:], self.shape)) or \
                builtins.any(b != 1 and a != b for a, b in zip(shape[new_dims:], self.shape)):
            raise ValueError("Non-broadcastable.")
        bd = [i < new_dims or (shape[i] != 1 and self.shape[i - new_dims] == 1) for i in range(len(shape))]
        if not self.bdarray.remote_constructed:
            DAG.instantiate(self)
        return ndarray(shape, base=self, distribution=shardview.broadcast(self.distribution, bd, shape),
                       local_border=0, readonly=True)

    def broadcastable_to(self, shape):
        new_dims = len(shape) - len(self.shape)
        if new_dims < 0:
            return False
        return not builtins.any(a > 1 and b > 1 and a != b for a, b in zip(shape[new_dims:], self.shape))

    def array_unaryop(self, op, optext, reduction=False, dtype=None, axis=None, keepdims=False, asarray=False, elide=None):
        if dtype is None:
            dtype = self.dtype
        elif isinstance(dtype, str) and dtype == "float":
            dtype = np.float32 if self.dtype == np.float32 else np.float64
        dtype = np.dtype(dtype)
        if not reduction:
            new = create_array_with_divisions(self.shape, self.distribution, dtype=dtype)
            DAG.assign(new, E(optext, self))
            return new
        return self._reduction(op, dtype, axis, keepdims, asarray, elide)

    def array_binop(self, rhs, op, optext, inplace=False, reverse=False, dtype=None):
        if isinstance(rhs, np.ndarray):
            rhs = fromarray(rhs) if rhs.shape != () else rhs.item()
        if isinstance(rhs, (list, tuple)):
            rhs = fromarray(np.array(rhs))
        if not isinstance(rhs, (ndarray, numbers.Number, np.generic, bool)):
            return NotImplemented
        new_dtype = unify_args(self.dtype, rhs, dtype)
        if op == "__truediv__":
            # division becomes multiplication by the reciprocal (ramba/ramba.py:6121-6126)
            op, optext = "__mul__", "mul"
            rhs = 1.0 / rhs
        elif op == "__itruediv__":
            op, optext = "__imul__", "mul"
            rhs = 1.0 / rhs
        new_shape, selfview, rhsview = ndarray.broadcast(self, rhs)
        if new_shape is None:  # 0-d with scalar: compute on the host
            a = self.distribution if isinstance(self, ndarray) else self
            b = rhs.distribution if isinstance(rhs, ndarray) else rhs
            res = getattr(np.asarray(a), op)(b) if not reverse else getattr(np.asarray(a), op)(b)
            return array(res)
        if inplace:
            if self.readonly:
                raise ValueError("assignment destination is read-only")
            assert self.shape == new_shape, "non-broadcastable output operand"
            DAG.assign(self, E(optext, self, rhsview))
            return self
        new = empty(new_shape, dtype=new_dtype)
        if reverse:
            DAG.assign(new, E(optext, rhsview, selfview))
        else:
            DAG.assign(new, E(optext, selfview, rhsview))
        return new

    # ---- reductions (ramba/ramba.py:5789-5937)
    def _reduction(self, op, dtype, axis, keepdims, asarray, elide=None):
        if axis is not None:
            if isinstance(axis, numbers.Number):
                axis = [axis]
            axis = sorted(a % self.ndim if -self.ndim <= a < self.ndim else _raise_axis(a, self.ndim) for a in axis)
            if len(axis) == self.ndim:
                axis = None
        red = REDUCTIONS[op]
        init = red.identity(dtype)
        src = self
        if red.truth:
            init = bool(init)  # (the partial array of all / any starts as a truth value)
            # reduce each element's truth value: a product or sum of 0/1 cannot wrap, underflow, reach NaN or cancel
            src = E("ne", self, 0)
        elif dtype_class(rb_dtype(dtype)) != dtype_class(rb_dtype(self.dtype)):
            src = E("astype", self, imm=rb_dtype(dtype))  # sum / prod(dtype=D): each element is converted to D first
        if self.maskarray is not None:
            axis = None
        if axis is None or (axis == [0] and self.ndim == 1):
            dsz, dist, bdist = shardview.reduce_all_axes(self.shape, self.distribution)
            red_arr = full(dsz, init, dtype=dtype, distribution=dist, no_defer=True)
            red_bcast = ndarray(self.shape, base=red_arr, distribution=bdist, local_border=0, readonly=False)
            DAG.reduce(op, src if self.maskarray is None else E("where", self.maskarray, src, red_identity(op, dtype)),
                       red_bcast, elide=elide)
            return _reduction2b(red_arr, op, dtype, asarray)
        dsz, dist, bdist = shardview.reduce_axes(self.shape, self.distribution, axis)
        red_arr = full(dsz, init, dtype=dtype, distribution=dist, no_defer=True)
        red_bcast = ndarray(self.shape, base=red_arr, distribution=bdist, local_border=0, readonly=False)
        DAG.reduce(op, src, red_bcast, axis, elide)
        return _reduction2(red_arr, op, dtype, axis, keepdims is True)

    def mean(self, axis=None, dtype=None, **kwargs):
        n = self.size if axis is None else int(np.prod([self.shape[a] for a in ([axis] if isinstance(axis, numbers.Number) else axis)]))
        # integer and bool data: NumPy's float64 sum of float64(x) (an integer sum would wrap, a bool sum is an `or`)
        s = self.sum(axis=axis, dtype=np.float64 if self.dtype.kind in "iub" else None, **kwargs)
        if dtype is None:
            dtype = np.float64 if self.dtype.kind in "iub" else self.dtype
        if isinstance(s, ndarray):
            return (s * (1.0 / n)).astype(dtype) if np.dtype(dtype) != np.result_type(s.dtype, 1.0) else s * (1.0 / n)
        return np.dtype(dtype).type(s / n)

    # ---- views
    @staticmethod
    def _plain_index(index):
        """Index as a tuple; 0-d arrays of an integer dtype index like the integer they hold
        (ramba/tests/test_distributed_array.py:712-752)."""
        if not isinstance(index, tuple):
            index = (index,)
        return tuple(int(i.distribution.item()) if isinstance(i, ndarray) and i.shape == () and i.dtype.kind in "iu" else i
                     for i in index)

    def __getitem__(self, index):
        if isinstance(index, ndarray) and index.dtype == np.bool_:
            if not index.broadcastable_to(self.shape):
                raise IndexError("Mask index shape does not match array shape")
            m = index if index.shape == self.shape else index.broadcast_to(self.shape)
            return ndarray(self.shape, base=self, distribution=self.distribution, local_border=0,
                           readonly=self.readonly, maskarray=m)
        index = self._plain_index(index)
        if advindex.has_advanced(index):
            return advindex.getitem(self, index)
        if builtins.any(i is None for i in index):
            # newaxis: slice without the None terms, then insert unit dims where they stood
            n_spec = builtins.sum(1 for i in index if i is not None and i is not Ellipsis)
            terms = []
            for i in index:
                if i is Ellipsis:
                    terms.extend([slice(None)] * (self.ndim - n_spec))
                else:
                    terms.append(i)
            sub = self[tuple(t for t in terms if t is not None)]
            if not isinstance(sub, ndarray):
                raise NotImplementedError("newaxis on a single element")
            axes, out_pos = [], 0
            for t in terms:
                if t is None:
                    axes.append(out_pos)
                    out_pos += 1
                elif isinstance(t, slice):
                    out_pos += 1
            return sub.expand_dims(tuple(axes))
        if builtins.any(i is Ellipsis for i in index):
            pos = [j for j, i in enumerate(index) if i is Ellipsis][0]
            fill = self.ndim - (len(index) - 1)
            index = index[:pos] + (slice(None),) * fill + index[pos + 1:]
        if self.shape == ():
            if len(index) != 0:
                raise IndexError("too many indices for array: array is 0-dimensional, but %d were indexed" % len(index))
            return self.distribution[()]
        if builtins.all(isinstance(i, numbers.Integral) for i in index) and len(index) == self.ndim:
            cindex = canonical_index(index, self.shape)
            DAG.instantiate(self)
            return getitem_global(self, tuple(s.start for s in cindex))
        if not self.bdarray.remote_constructed:
            DAG.instantiate(self)
        # the partition of a slice view is a pure function of (this view's distribution, the index): computed once per
        # array and index - an iterative program takes the same slices every step (ramba/ramba.py:6548-6579 recomputes)
        try:
            key = tuple((i.start, i.stop, i.step) if type(i) is slice else ("i", int(i)) for i in index)
            hit = self._slices.get(key) if self._slices is not None else None
        except TypeError:
            key, hit = None, None
        if hit is None:
            cindex = canonical_index(index, self.shape)
            dim_shapes = tuple(_slice_len(x) for x in cindex)
            sdist = shardview.slice_distribution(cindex, self.distribution)
            axismap = [i for i in range(len(dim_shapes)) if i >= len(index) or isinstance(index[i], slice)]
            if len(axismap) < len(dim_shapes):
                dim_shapes, sdist = shardview.remap_axis(dim_shapes, sdist, axismap)
            hit = (dim_shapes, sdist)
            if key is not None:
                if self._slices is None:
                    self._slices = {}
                if len(self._slices) < 64:
                    self._slices[key] = hit
        dim_shapes, sdist = hit
        return ndarray(dim_shapes, base=self, distribution=sdist, local_border=0, readonly=self.readonly)

    def __setitem__(self, index, value):
        if self.readonly:
            raise ValueError("assignment destination is read-only")
        if isinstance(value, (list, tuple)):
            value = np.array(value)
        if self.shape == ():  # 0-d arrays keep their value on the host (like the reference)
            if self._plain_index(index) not in ((), (Ellipsis,)):
                raise IndexError("too many indices for array: array is 0-dimensional")
            self.distribution[()] = value.distribution.item() if isinstance(value, ndarray) else value
            return
        if not (isinstance(index, ndarray) and index.dtype == np.bool_):
            index = self._plain_index(index)
            if advindex.has_advanced(index):
                advindex.setitem(self, index, value)
                return
            if builtins.any(i is Ellipsis for i in index) and not builtins.any(i is None for i in index):
                pos = [j for j, i in enumerate(index) if i is Ellipsis][0]
                index = index[:pos] + (slice(None),) * (self.ndim - (len(index) - 1)) + index[pos + 1:]
        view = self[index]
        if not isinstance(view, ndarray):  # single element
            cindex = canonical_index(index, self.shape)
            view = self[tuple(slice(s.start, s.start + 1) for s in cindex)]
        if isinstance(value, np.ndarray):
            while value.ndim > view.ndim and value.shape[0] == 1:  # NumPy drops extra leading unit dims of the value
                value = value[0]
            if value.size == 1:
                value = value.reshape(())
        if isinstance(value, (numbers.Number, np.generic)) or (isinstance(value, np.ndarray) and value.shape == ()):
            DAG.assign(view, value if not isinstance(value, np.ndarray) else value.item())
            return
        if isinstance(value, np.ndarray):
            value = fromarray(value)
        if value.shape == ():
            DAG.assign(view, value.distribution.item())
            return
        if not value.broadcastable_to(view.shape):
            raise ValueError("could not broadcast input array from shape %s into shape %s" % (value.shape, view.shape))
        if value.shape != view.shape:
            value = value.broadcast_to(view.shape)
        if not (view.gid == value.gid and shardview.dist_is_eq(view.distribution, value.distribution)):
            DAG.assign(view, value)

    def remapped_axis(self, newmap):
        if not self.bdarray.remote_constructed:
            DAG.instantiate(self)
        newshape, newdist = shardview.remap_axis(self.shape, self.distribution, newmap)
        return ndarray(newshape, base=self, distribution=newdist, local_border=0, readonly=self.readonly)

    def expand_dims(self, axis):
        axes = (axis,) if isinstance(axis, numbers.Integral) else tuple(axis)
        k = self.ndim + len(axes)
        axes = sorted(a % k for a in axes)
        if len(set(axes)) != len(axes):
            raise ValueError("repeated axis")
        if not self.bdarray.remote_constructed:
            DAG.instantiate(self)
        newshape, newdist = shardview.expand_unit_dims(self.shape, self.distribution, axes)
        return ndarray(newshape, base=self, distribution=newdist, local_border=0, readonly=True)

    def squeeze(self, axis=None):
        if axis is None:
            axes = tuple(i for i in range(self.ndim) if self.shape[i] == 1)
        else:
            axes = tuple(a % self.ndim for a in ((axis,) if isinstance(axis, numbers.Integral) else tuple(axis)))
        if not builtins.all(self.shape[a] == 1 for a in axes):
            raise ValueError("cannot select an axis to squeeze out which has size not equal to one")
        return self.remapped_axis([i for i in range(self.ndim) if i not in axes])

    def reshape(self, *shape):
        """Reshapes that insert or remove unit dims are views; anything else has to move data between shards and, like in the
        reference (ramba/ramba.py:9178-9238), raises ReshapeError unless RAMBA_RESHAPE_COPY forwards it to reshape_copy."""
        if len(shape) == 1 and isinstance(shape[0], (tuple, list)):
            shape = tuple(shape[0])
        shape = _norm_newshape(self, shape)
        if shape == self.shape:
            return self
        if [s for s in shape if s != 1] != [s for s in self.shape if s != 1]:
            if common.reshape_forwarding:
                return reshape_copy(self, shape)
            raise ReshapeError(
                "ramba.reshape not supported as distributed array reshape cannot be done inplace.  Use reshape_copy instead to "
                "create a non-inplace reshape or set RAMBA_RESHAPE_COPY environment variable to convert all reshape calls to "
                "reshape_copy.")
        flat = self.squeeze() if builtins.any(s == 1 for s in self.shape) else self
        axes = [i for i, s in enumerate(shape) if s == 1]
        return flat.expand_dims(axes) if axes else flat

    def reshape_copy(self, newshape):
        return reshape_copy(self, newshape)

    def transpose(self, *args):
        nd = self.ndim
        if len(args) == 0 or (len(args) == 1 and args[0] is None):
            return self.remapped_axis(list(range(nd - 1, -1, -1)))
        if len(args) == 1 and isinstance(args[0], (tuple, list)):
            args = tuple(args[0])
        axes = [a % nd for a in args]
        if sorted(axes) != list(range(nd)):
            raise ValueError("axes don't match array")
        return self.remapped_axis(axes)

    def swapaxes(self, a1, a2):
        axes = list(range(self.ndim))
        axes[a1], axes[a2] = axes[a2], axes[a1]
        return self.remapped_axis(axes)

    def moveaxis(self, source, destination):
        src = [s % self.ndim for s in ([source] if isinstance(source, numbers.Integral) else list(source))]
        dst = [d % self.ndim for d in ([destination] if isinstance(destination, numbers.Integral) else list(destination))]
        order = [n for n in range(self.ndim) if n not in src]
        for d, s in sorted(zip(dst, src)):
            order.insert(d, s)
        return self.remapped_axis(order)

    def astype(self, dtype, copy=True):
        dtype = np.dtype(dtype)
        if dtype == self.dtype:
            return globals()["copy"](self) if copy else self
        new = create_array_with_divisions(self.shape, self.distribution, dtype=dtype)
        DAG.assign(new, self)
        return new

    def clip(self, a_min, a_max, out=None):
        new = out if out is not None else create_array_with_divisions(self.shape, self.distribution, dtype=self.dtype)
        DAG.assign(new, E("min", a_max, E("max", self, a_min)))
        return new

    def allclose(self, other, rtol=1e-5, atol=1e-8, equal_nan=False):
        return bool(isclose(self, other, rtol=rtol, atol=atol, equal_nan=equal_nan).all())

    def isclose(self, other, rtol=1e-5, atol=1e-8, equal_nan=False):
        return isclose(self, other, rtol=rtol, atol=atol, equal_nan=equal_nan)

    def nansum(self, asarray=False, **kwargs):
        """Sum of the elements that are not NaN (ramba/ramba.py:6777-6781: a masked sum)."""
        v = self[isnan(self).logical_not()].sum(asarray=True, **kwargs)  # noqa: F821
        return v if asarray else v[0]

    def nanmean(self, axis=None, dtype=None):
        """Mean of the elements that are not NaN (whole array, like the reference: ramba/ramba.py:6766-6772)."""
        assert axis is None, "nanmean over an axis is not implemented (nor by the reference, ramba/ramba.py:6760-6763)"
        ok = isnan(self).logical_not()  # noqa: F821
        s = self[ok].sum(dtype=np.float64 if self.dtype.kind in "iub" else None)  # (as in mean)
        return s / ok.astype(np.int64).sum()  # (a bool sum stays bool, like in the reference)

    def rollaxis(self, axis, start=0):
        """NumPy's rollaxis (ramba/ramba.py:5643-5654)."""
        nd = self.ndim
        if not -nd <= axis < nd:
            raise np.exceptions.AxisError(axis, nd)
        axis %= nd
        if not isinstance(start, numbers.Integral):
            raise TypeError("integer argument expected")
        if start < -nd or start > nd:
            raise np.exceptions.AxisError("`start` arg requires %d <= start < %d but %d was passed in" % (-nd, nd + 1, start))
        if start < 0:
            start += nd
        if start > axis:
            start -= 1
        return self.moveaxis(axis, start)

    # ---- NumPy protocol hooks (ramba/ramba.py:6825-6894)
    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        if method != "__call__" or kwargs.get("out") is not None:
            return NotImplemented
        name = ufunc.__name__
        alias = {"multiply": "mul", "subtract": "sub", "divide": "truediv", "true_divide": "truediv",
                 "floor_divide": "floordiv", "add": "add", "power": "pow", "remainder": "mod", "mod": "mod",
                 "absolute": "abs", "negative": "neg", "greater": "gt", "less": "lt", "greater_equal": "ge",
                 "less_equal": "le", "equal": "eq", "not_equal": "ne", "bitwise_and": "and", "bitwise_or": "or",
                 "bitwise_xor": "xor", "left_shift": "lshift", "right_shift": "rshift", "invert": "invert"}
        name = alias.get(name, name)
        if len(inputs) == 1:
            f = getattr(self, name, None) or getattr(self, "__" + name + "__", None)
            return f() if f is not None else NotImplemented
        a, b = inputs
        if a is self:
            f = getattr(self, "__" + name + "__", None) or getattr(self, name, None)
            return f(b) if f is not None else NotImplemented
        f = getattr(self, "__r" + name + "__", None)
        if f is not None:
            return f(a)
        if name in ("gt", "lt", "ge", "le", "eq", "ne"):
            swap = {"gt": "lt", "lt": "gt", "ge": "le", "le": "ge", "eq": "eq", "ne": "ne"}[name]
            return getattr(self, "__" + swap + "__")(a)
        f = getattr(self, name, None)  # commutative named ops (minimum, maximum, logical_*)
        return f(a) if f is not None else NotImplemented

    def __array_function__(self, func, types, args, kwargs):
        f = HANDLED_FUNCTIONS.get(func.__name__)
        if f is None:
            return NotImplemented
        return f(*args, **kwargs)


def _raise_axis(a, nd):
    raise np.exceptions.AxisError(a, nd)


def _local_partial_tensor(red_arr, n, op):
    """This rank's block of the partial array as a flat device tensor of n elements in the accumulator dtype (float64 /
    int64) - the reduction's identity when the rank holds no part."""
    w = common.worker_num
    acc_dt = torch.float64 if red_arr.dtype.kind == "f" else torch.int64
    sv = red_arr.distribution[w]
    sh = blocks.block(red_arr)
    if shardview.is_empty(sv):
        return torch.full((n,), red_identity(op, red_arr.dtype), dtype=acc_dt, device=RT.device)
    return sh.interior().reshape(-1)[:n].to(acc_dt)


_KEY_FLIP = 0x7FFFFFFFFFFFFFFF


def _all_reduce_partials(t, op):
    """t = op over every rank's partials, in place.  Float min / max reduce order-preserving int64 keys of the float64
    bits with NaN beyond every number, so a NaN on any rank wins (NumPy) whatever the backend's float MIN / MAX do with
    NaN; one collective, as for sum."""
    if op not in ("min", "max") or not t.is_floating_point():
        RT.all_reduce(t, op)
        return
    nan_key = torch.iinfo(torch.int64).min if op == "min" else torch.iinfo(torch.int64).max
    bits = t.view(torch.int64)
    key = torch.where(bits < 0, bits ^ _KEY_FLIP, bits)
    key = torch.where(torch.isnan(t), nan_key, key)
    RT.all_reduce(key, op)
    val = torch.where(key < 0, key ^ _KEY_FLIP, key).view(torch.float64)
    t.copy_(torch.where(key == nan_key, float("nan"), val))


def _reduction2b(red_arr, op, dtype, asarray):
    """Stage 2 of a global reduction.  The reference gathers one partial per worker to the driver and reduces them
    there (ramba/ramba.py:5852-5863); under SPMD every rank needs the result, so the partials (one element per rank,
    on the GPUs) are combined by ONE all-reduce and only the scalar comes back to the host."""
    if builtins.all(i == 1 for i in red_arr.shape):
        if not asarray and common.num_workers == 1:
            # one rank, one partial: read it straight from the shard (same value and type as indexing the array)
            DAG.instantiate(red_arr)
            return _part_to_host(red_arr, 0).reshape(-1)[0]
        sl = (0,) * red_arr.ndim if not asarray else (slice(0, 1),) + (0,) * (red_arr.ndim - 1)
        return red_arr[sl]
    if common.num_workers > 1:
        DAG.instantiate(red_arr)
        t = _local_partial_tensor(red_arr, 1, op)
        _all_reduce_partials(t, op)
        val = t.cpu().numpy()[0]
        if REDUCTIONS[op].truth:
            val = np.bool_(val != 0)
    else:
        local = np.array(red_arr.asarray())
        val = getattr(np, op)(local)  # (NumPy names its reductions the same)
    if not asarray:
        return np.sum(val, dtype=dtype)
    return full((1,), val, dtype=dtype)


def _split_only_along(red_arr, axis):
    """True when every rank's block of the partial array spans the kept axes completely (the source array is cut along
    reduced axes only), so that stage 2 is an element-wise combination of whole partial rows."""
    for sv in red_arr.distribution:
        if shardview.is_empty(sv):
            continue
        for d in range(red_arr.ndim):
            if d in axis:
                if int(sv.size[d]) != 1:
                    return False
            elif int(sv.start[d]) != 0 or int(sv.size[d]) != red_arr.shape[d]:
                return False
    return True


def _reduction2(red_arr, op, dtype, axis, keepdims):
    """Stage 2 of an axis reduction: fold the per-division partial slices (ramba/ramba.py:5818-5849).  When the
    partial rows live on different ranks and each rank holds whole rows, they are summed by ONE all-reduce (each rank
    then keeps its own division of the result); otherwise a second fused op over the partial slices does it."""
    nd = red_arr.ndim
    if keepdims:
        sl1 = tuple(slice(None) for _ in range(nd))
    else:
        sl1 = tuple(0 if i in axis else slice(None) for i in range(nd))
    sl2 = tuple(slice(0, 1) if i in axis else slice(None) for i in range(nd))
    k = [red_arr.shape[a] for a in axis]
    if builtins.all(x == 1 for x in k):
        return red_arr if keepdims else red_arr[sl1]
    kept_elems = int(np.prod([red_arr.shape[d] for d in range(nd) if d not in axis]))
    if common.num_workers > 1 and kept_elems <= (1 << 24) and _split_only_along(red_arr, axis):
        DAG.instantiate(red_arr)
        w = common.worker_num
        t = _local_partial_tensor(red_arr, kept_elems, op)
        _all_reduce_partials(t, op)
        out_shape = tuple(1 if d in axis else red_arr.shape[d] for d in range(nd))
        arr = ndarray(out_shape, dtype=red_arr.dtype, flex_dist=False)
        sh = blocks.block(arr)
        sv = arr.distribution[w]
        if not shardview.is_empty(sv):
            mine = t.view(out_shape)[shardview.to_slice(sv)]
            sh.interior().copy_(mine)  # (converts the accumulator dtype back to the array's)
        return arr if keepdims else arr[sl1]
    arr = empty_like(red_arr[sl2])
    combine = REDUCTIONS[op].combine
    expr = None
    for j in np.ndindex(tuple(k)):
        sl = []
        ii = 0
        for i in range(nd):
            if i in axis:
                sl.append(slice(j[ii], j[ii] + 1))
                ii += 1
            else:
                sl.append(slice(None))
        piece = red_arr[tuple(sl)]
        expr = piece if expr is None else fold_expr(combine, expr, piece)
    DAG.assign(arr, expr)
    return arr[sl1]


# ---- operator tables (ramba/ramba.py:7893-7993) ------------------------------------------------
def _make_binop(name, optext, dtype=None, inplace=False, reverse=False):
    def _method(self, rhs):
        return self.array_binop(rhs, name, optext, inplace=inplace, reverse=reverse, dtype=dtype)

    _method.__name__ = name
    return _method


array_binop_funcs = {
    "__add__": ("add", None), "__mul__": ("mul", None), "__sub__": ("sub", None), "__floordiv__": ("floordiv", None),
    "__truediv__": ("div", "float"), "__mod__": ("mod", None), "__pow__": ("pow", None),
    "minimum": ("min", None), "maximum": ("max", None),
    "__gt__": ("gt", np.bool_), "__lt__": ("lt", np.bool_), "__ge__": ("ge", np.bool_), "__le__": ("le", np.bool_),
    "__eq__": ("eq", np.bool_), "__ne__": ("ne", np.bool_),
    "logical_and": ("land", np.bool_), "logical_or": ("lor", np.bool_), "logical_xor": ("lxor", np.bool_),
    "__and__": ("band", None), "__xor__": ("bxor", None), "__or__": ("bor", None),
    "__lshift__": ("shl", None), "__rshift__": ("shr", None),
}
for _n, (_t, _d) in array_binop_funcs.items():
    setattr(ndarray, _n, _make_binop(_n, _t, dtype=_d))
array_binop_rfuncs = {
    "__radd__": ("add", None), "__rmul__": ("mul", None), "__rsub__": ("sub", None), "__rtruediv__": ("div", "float"),
    "__rfloordiv__": ("floordiv", None), "__rmod__": ("mod", None), "__rpow__": ("pow", None),
    "__rand__": ("band", None), "__rxor__": ("bxor", None), "__ror__": ("bor", None),
}
for _n, (_t, _d) in array_binop_rfuncs.items():
    setattr(ndarray, _n, _make_binop(_n, _t, dtype=_d, reverse=True))
array_inplace_binop_funcs = {
    "__iadd__": "add", "__isub__": "sub", "__imul__": "mul", "__itruediv__": "div", "__ifloordiv__": "floordiv",
    "__imod__": "mod", "__ipow__": "pow",
}
for _n, _t in array_inplace_binop_funcs.items():
    setattr(ndarray, _n, _make_binop(_n, _t, inplace=True))


def _ndarray_groupby(self, dim, value_to_group, num_groups=None):
    """Group the positions of axis `dim` by the integer labels `value_to_group` (ramba/ramba.py:6896-6899): a RambaGroupby
    whose sum / prod / min / max / count / mean / nanmean / var / std reduce every group on the grouped-reduction kernel
    (ramba_b200/groupby.py).  num_groups=None means value_to_group.max() + 1."""
    from .groupby import RambaGroupby

    return RambaGroupby(self, dim, value_to_group, num_groups)


ndarray.groupby = _ndarray_groupby
from . import groupby as _groupby_module  # noqa: E402

_groupby_module._install_binops(list(array_binop_funcs) + list(array_binop_rfuncs))
ndarray.__hash__ = None


def _make_unop(name, optext, dtype=None):
    def _method(self, **kwargs):
        if "dtype" not in kwargs:
            kwargs["dtype"] = dtype
        return self.array_unaryop(name, optext, **kwargs)

    _method.__name__ = name
    return _method


array_unaryop_funcs = {
    "__abs__": ("abs", None), "abs": ("abs", None), "square": ("square", None), "sqrt": ("sqrt", "float"),
    "sin": ("sin", "float"), "cos": ("cos", "float"), "tan": ("tan", "float"), "sinh": ("sinh", "float"),
    "cosh": ("cosh", "float"), "tanh": ("tanh", "float"), "arcsin": ("asin", "float"), "arccos": ("acos", "float"),
    "arctan": ("atan", "float"), "__neg__": ("neg", None), "exp": ("exp", "float"), "log": ("log", "float"),
    "cbrt": ("cbrt", "float"),
    "isfinite": ("isfinite", np.bool_), "isinf": ("isinf", np.bool_), "isnan": ("isnan", np.bool_),
    "isneginf": ("isneginf", np.bool_), "isposinf": ("isposinf", np.bool_), "logical_not": ("lnot", np.bool_),
    "__invert__": ("invert", None),
}
for _n, (_t, _d) in array_unaryop_funcs.items():
    setattr(ndarray, _n, _make_unop(_n, _t, dtype=_d))


def _make_reduction(name, dtype=None):
    def _method(self, axis=None, dtype=dtype, keepdims=False, asarray=False, **kwargs):
        # `(X*2.0 + 1.0).sum()`: the operand is a temporary that nobody can observe once this call returns.  The global
        # reduction flushes INSIDE the call, while the caller's expression still holds the temporary, so the reference
        # materialises it (ramba/ramba.py:8123-8127 looks at handle liveness only); here a temporary whose only
        # reference is the pending call is treated as already dead and never touches HBM.
        elide = None
        if _sys_getrefcount(self) <= _TEMP_REFCOUNT and self.base is None and self.bdarray.nrefs == 1 \
                and not self.bdarray.remote_constructed:
            elide = self.gid  # (add_op honours it only if the statement writing the temporary shares the fused op)
        return self.array_unaryop(name, None, reduction=True, dtype=dtype, axis=axis, keepdims=keepdims, asarray=asarray,
                                  elide=elide)

    _method.__name__ = name
    return _method


from sys import getrefcount as _sys_getrefcount  # noqa: E402


def _measure_temp_refcount():
    """Reference count a method sees for `self` when it is called on a temporary (CPython: the frame's own
    reference + getrefcount's argument).  Measured, not assumed: if the interpreter counts differently the
    elision simply never triggers."""
    class _Probe:
        pass

    def _method(self, axis=None, dtype=None, keepdims=False, asarray=False, **kwargs):
        return _sys_getrefcount(self)

    _Probe.m = _method
    temp = _Probe().m()
    named_obj = _Probe()
    named = named_obj.m()
    return temp if named > temp else -1


_TEMP_REFCOUNT = _measure_temp_refcount()


array_simple_reductions = {"sum": None, "prod": None, "min": None, "max": None, "all": np.bool_, "any": np.bool_}  # -> default dtype
for _n, _d in array_simple_reductions.items():
    setattr(ndarray, _n, _make_reduction(_n, _d))


# =============================================================================================
# host <-> device edges
# =============================================================================================
def _is_whole_shard(sv, sh):
    k = len(sv.size)
    return (k == len(sh.shape) and builtins.all(int(sv.axis_map[d]) == d and int(sv.steps[d]) == 1 and int(sv.base_offset[d]) == 0
                                                and int(sv.size[d]) == sh.shape[d] for d in range(k)))


def _part_to_host(nd, w, out=None, non_blocking=False):
    """This worker's part of view `nd` as a contiguous host array (get_view, ramba/ramba.py:2160-2176)."""
    if nd.bdarray.failed is not None:
        _raise_failed(nd.bdarray)
    sv = nd.distribution[w]
    sh = blocks.block(nd)  # (on every rank, also where the part is empty: the partition is fixed everywhere or nowhere)
    if shardview.is_empty(sv):
        return np.zeros([0] * nd.ndim, dtype=nd.dtype)
    shape = [int(x) for x in sv.size]
    if _is_whole_shard(sv, sh) and sh.border == 0 and nd.dtype != np.bool_:
        n = int(np.prod(shape))
        if out is not None and out.flags.c_contiguous and out.dtype == nd.dtype and out.size == n:
            # straight DMA (pinned `out`: full PCIe rate)
            torch.from_numpy(out.reshape(-1)).copy_(sh.buf[:n], non_blocking=non_blocking)
            return out.reshape(shape)
        t = sh.buf[:n]
        host = t.cpu()
        if host.data_ptr() == t.data_ptr():
            host = host.clone()  # (a host-resident shard: the caller gets a copy, never an alias of the live block)
        return host.numpy().reshape(shape)
    cst, n = _contig_strides(shape)
    buf = torch.empty(max(n, 1), dtype=torch_dtype(nd.dtype), device=RT.device)
    ptr, st, _, _ = blocks.part(nd)
    code = rb_dtype(nd.dtype)
    RT.launch(_pack_program(code, code), shape, [0] * len(shape),
              [(ptr, st, code), (buf.data_ptr(), cst, code)])
    RT.synchronize()
    host = buf[:n].cpu().numpy().reshape(shape)
    if nd.dtype == np.bool_:
        host = host.astype(np.bool_)
    return host


def gather_to_host(nd, out=None, non_blocking=False):
    """Full NumPy copy of a distributed view on every rank (asarray, ramba/ramba.py:5735-5765)."""
    w, W = common.worker_num, common.num_workers
    if W == 1:
        sv = nd.distribution[0]
        if shardview.is_empty(sv):
            return np.empty(nd.shape, dtype=nd.dtype) if out is None else out
        mine = _part_to_host(nd, w, out=out, non_blocking=non_blocking)
        if tuple(mine.shape) == tuple(nd.shape):
            return mine
        ret = np.empty(nd.shape, dtype=nd.dtype) if out is None else out
        ret[shardview.to_slice(sv)] = mine
        return ret
    ret = np.empty(nd.shape, dtype=nd.dtype) if out is None else out
    mine = _part_to_host(nd, w)
    store_dt = np.dtype(np.uint8) if nd.dtype == np.bool_ else nd.dtype
    for i in range(W):
        sv = nd.distribution[i]
        if shardview.is_empty(sv):
            continue
        shape = [int(x) for x in sv.size]
        nbytes = int(np.prod(shape)) * store_dt.itemsize
        # collectives move raw bytes: not every backend knows uint16/uint32
        if i == w:
            host = np.ascontiguousarray(mine.astype(np.uint8) if nd.dtype == np.bool_ else mine)
            t = torch.from_numpy(host.view(np.uint8).reshape(-1))
        else:
            t = torch.empty(nbytes, dtype=torch.uint8)
        t = t.to(RT.device)
        RT.broadcast(t, i)
        part = t.cpu().numpy().view(store_dt).reshape(shape)
        if nd.dtype == np.bool_:
            part = part.astype(np.bool_)
        ret[shardview.to_slice(sv)] = part
    return ret


def getitem_global(nd, index):
    """One element as a NumPy scalar (getitem_global, ramba/ramba.py:2183-2189)."""
    sl = tuple(slice(i, i + 1) for i in index)
    v = nd[sl]
    return gather_to_host(v).reshape(-1)[0]


def fromarray(x, local_border=0, dtype=None, **kwargs):
    """Distribute a NumPy array: every rank uploads its own block (ramba/ramba.py:8785-8850)."""
    if isinstance(x, numbers.Number):
        return array(x)
    x = np.asarray(x)
    if dtype is None:
        dtype = x.dtype
    if x.shape == ():
        return array(x.astype(dtype))
    new = ndarray(x.shape, dtype=dtype, flex_dist=False, local_border=local_border, **kwargs)
    deferred_op.do_ops()
    sv = new.distribution[common.worker_num]
    sh = blocks.block(new)
    if not shardview.is_empty(sv):
        blk = x[shardview.to_slice(sv)]
        if blk.dtype != new.dtype:
            blk = blk.astype(new.dtype)
        if not blk.flags.c_contiguous:
            blk = np.ascontiguousarray(blk)
        if new.dtype == np.bool_:
            blk = blk.astype(np.uint8)
        t = torch.from_numpy(blk.reshape(-1))  # a view when x is contiguous: pinned x -> straight DMA
        if sh.border:
            sh.interior().copy_(t.view(sh.shape), non_blocking=True)
        else:
            sh.buf[: t.numel()].copy_(t, non_blocking=True)
    return new


def fromarray_local(block, shape, dtype=None, **kwargs):
    """SPMD extension (no reference counterpart): every rank supplies ITS OWN block of a global
    array of shape `shape` (block shape = this rank's division under the default distribution).
    Used when the global array never exists on one host (bench.py's multi-GPU e2e leg)."""
    block = np.asarray(block)
    if dtype is None:
        dtype = block.dtype
    new = ndarray(shapeToInt(shape), dtype=dtype, flex_dist=False, **kwargs)
    deferred_op.do_ops()
    sv = new.distribution[common.worker_num]
    sh = blocks.block(new)
    if not shardview.is_empty(sv):
        if tuple(block.shape) != tuple(int(x) for x in sv.size):
            raise ValueError("fromarray_local: block shape %s != this rank's division %s" % (block.shape, tuple(int(x) for x in sv.size)))
        blk = block if block.dtype == new.dtype else block.astype(new.dtype)
        if not blk.flags.c_contiguous:
            blk = np.ascontiguousarray(blk)
        if new.dtype == np.bool_:
            blk = blk.astype(np.uint8)
        t = torch.from_numpy(blk.reshape(-1))
        if sh.border:
            sh.interior().copy_(t.view(sh.shape), non_blocking=True)
        else:
            sh.buf[: t.numel()].copy_(t, non_blocking=True)
    return new


def load(fname, dtype=None, local=False, ftype=None, **kwargs):
    """Array from a file (ramba/ramba.py:8930-8945).  File types that can be read in parts are loaded DISTRIBUTED: every rank
    reads only the block of the file its shard holds (the worker side of the reference, RemoteState.load 3929-3956) and
    uploads it; the others (images) are read whole and distributed like `fromarray`.  `local=True` forces the second way.
    Extra keyword arguments go to the handler (`arr_path` for HDF5, `var_select` for netCDF)."""
    from . import fileio

    fldr = fileio.get_load_handler(fname, ftype)
    if local or not fldr.is_dist:
        tmp = fldr.readall(fname, **kwargs)
        return fromarray(tmp, dtype=tmp.dtype if dtype is None else dtype)
    shp, dt = fldr.getinfo(fname, **kwargs)
    shp = shapeToInt(shp)
    if dtype is None:
        dtype = dt
    if shp == ():
        return array(np.asarray(fldr.readall(fname, **kwargs)).astype(dtype))
    sv = shardview.default_distribution(shp)[common.worker_num]
    if shardview.is_empty(sv):
        block = np.empty([0] * len(shp), dtype=dtype)
    else:
        block = fldr.read(fname, shardview.to_slice(sv), **kwargs)
    return fromarray_local(block, shp, dtype=dtype)


def local_block_to_host(nd, out=None, non_blocking=False):
    """SPMD extension: this rank's block of `nd` as a host array (no gather)."""
    DAG.instantiate(nd)
    return _part_to_host(nd, common.worker_num, out=out, non_blocking=non_blocking)


def array(x, dtype=None, copy=True, **kwargs):
    if isinstance(x, ndarray):
        return x.copy() if copy else x
    a = np.array(x, dtype=dtype)
    if a.shape == ():
        if dtype is None:
            a = a.astype(np.float64)  # 0-d arrays default to float64 like every array of the reference (ramba/ramba.py:8831-8837)
        nd = ndarray((), dtype=a.dtype)
        nd.distribution = a
        nd.bdarray.distribution = a
        return nd
    return fromarray(a, **kwargs)


def asarray(x, dtype=None, **kwargs):
    if isinstance(x, ndarray):
        return x if dtype is None or np.dtype(dtype) == x.dtype else x.astype(dtype)
    return array(x, dtype=dtype)


# =============================================================================================
# creation (ramba/ramba.py:8563-8991)
# =============================================================================================
def create_array_with_divisions(shape, divisions, local_border=0, dtype=None):
    # (a new array given a partition gets the same boxes with fresh buffer coordinates: assign_bdarray cleans it)
    return ndarray(shape, dtype=dtype, distribution=divisions, local_border=local_border, flex_dist=False)


def create_array(shape, filler, local_border=0, dtype=None, distribution=None, no_defer=False, **kwargs):
    shape = shapeToInt(shape)
    if dtype is None:
        dtype = np.float64
    new = ndarray(shape, dtype=dtype, distribution=distribution, local_border=local_border,
                  flex_dist=(distribution is None), **kwargs)
    if shape == ():
        new.distribution = np.array(0 if filler is None else filler, dtype=dtype)
        new.bdarray.distribution = new.distribution
        return new
    if filler is None:
        return new  # allocation is lazy; nothing to run (empty)
    if no_defer:
        # out-of-band creation: allocate and fill now WITHOUT flushing the pending fused op, so that
        # the producers of a reduction stay fused with it (ramba/ramba.py:5918, 8603-8627)
        _fill_now(new, filler)
        return new
    DAG.assign(new, filler)
    return new


_fill_programs = {}


def _fill_now(nd, value):
    """Fill this worker's block of a brand-new array with a scalar, immediately."""
    sv = nd.bdarray.distribution[common.worker_num]
    sh = blocks.block(nd)
    if shardview.is_empty(sv):
        return
    code = rb_dtype(nd.dtype)
    if isinstance(value, np.generic):
        value = value.item()
    key = (code, type(value), value)
    prog = _fill_programs.get(key)
    if prog is None:
        lw = Lowering([code])
        lw.store(0, lw.scalar(value))
        prog = _fill_programs[key] = lw.finish()
    n = sh.buf.numel()  # (the ring of a padded block is filled too)
    RT.launch(prog, [n], [0], [(sh.buf.data_ptr(), [1], code)])


def init_array(shape, filler, local_border=0, dtype=None, distribution=None, tuple_arg=True, **kwargs):
    """Array filled by `filler`: a constant, or a function of the global index - which it receives as ONE tuple
    unless tuple_arg is False (ramba/ramba.py:8658-8676; fromfunction is the tuple_arg=False form, 8904-8905)."""
    if callable(filler):
        if isinstance(shape, numbers.Integral):
            shape = (shape,)
        return fromfunction((lambda *idx: filler(idx)) if tuple_arg else filler, shape, dtype=dtype)
    return create_array(shape, filler, local_border=local_border, dtype=dtype, distribution=distribution, **kwargs)


def empty(shape, dtype=None, order="C", local_border=0, distribution=None, **kwargs):
    return create_array(shape, None, local_border=local_border, dtype=dtype, distribution=distribution, **kwargs)


def empty_like(other, dtype=None, **kwargs):
    return empty(other.shape, dtype=other.dtype if dtype is None else dtype, **kwargs)


def zeros(shape, dtype=None, order="C", local_border=0, distribution=None, **kwargs):
    return create_array(shape, 0, local_border=local_border, dtype=dtype, distribution=distribution, **kwargs)


def zeros_like(other, dtype=None, shape=None, **kwargs):
    return zeros(other.shape if shape is None else shape, dtype=other.dtype if dtype is None else dtype)


def ones(shape, dtype=None, order="C", local_border=0, distribution=None, **kwargs):
    return create_array(shape, 1, local_border=local_border, dtype=dtype, distribution=distribution, **kwargs)


def ones_like(other, dtype=None, shape=None, **kwargs):
    return ones(other.shape if shape is None else shape, dtype=other.dtype if dtype is None else dtype)


def full(shape, v, dtype=None, local_border=0, **kwargs):
    """Constant fill.  Like every creation routine of the reference the dtype defaults to float64 whatever the
    fill value is (ramba/ramba.py:8753-8754 -> init_array -> bdarray default, 1125-1126)."""
    return create_array(shape, v, local_border=local_border, dtype=np.float64 if dtype is None else dtype, **kwargs)


def _full_of(shape, v):
    """Constant array in the value's own dtype (internal: scalar results of traced user functions)."""
    return create_array(shape, v, dtype=np.asarray(v).dtype)


def full_like(other, v, dtype=None, **kwargs):
    return full(other.shape, v, dtype=other.dtype if dtype is None else dtype)


def copy(arr, local_border=0):
    new = create_array_with_divisions(arr.shape, arr.distribution, dtype=arr.dtype)
    DAG.assign(new, arr)
    return new


def arange(start, stop=None, step=None, dtype=None, *, like=None, local_border=0):
    """index[0] + global_start[0] as a fused op (ramba/ramba.py:8952-8972)."""
    if stop is None:
        size = start
    elif step is None:
        size = stop - start
    else:
        size = (stop - start + step - 1) // step
    res = empty((builtins.max(0, int(size)),), dtype=np.int64 if dtype is None else dtype, local_border=local_border)
    if stop is None:
        expr = Iota(0)
    elif step is None:
        expr = E("add", start, Iota(0))
    else:
        expr = E("add", start, E("mul", step, Iota(0)))
    DAG.assign(res, expr)
    return res


def linspace(start, stop, num=50, endpoint=True, retstep=False, dtype=None):
    assert num > 0
    length = stop - start
    step = length / (num - 1) if endpoint else length / num
    res = arange(num) * step + start
    if dtype is not None:
        res = res.astype(dtype)
    return (res, step) if retstep else res


def fromfunction(function, shape, dtype=None, **kwargs):
    """Index-driven filler.  The reference compiles `function` with Numba per element
    (ramba/ramba.py:1535-1595, 8904-8905); here it is evaluated ONCE on lazy index arrays
    (iota operands), so it must be built from array operators / ramba functions."""
    shape = shapeToInt(shape)
    if dtype is None:
        dtype = np.float64  # the reference's default array dtype (bdarray.assign_bdarray, ramba/ramba.py:1125-1126)
    idx = []
    for d in range(len(shape)):
        a = empty(shape, dtype=np.int64)
        DAG.assign(a, Iota(d))
        idx.append(a)
    out = function(*idx)
    if not isinstance(out, ndarray):
        out = _full_of(shape, out)
    if np.dtype(dtype) != out.dtype:
        out = out.astype(dtype)
    return out


def eye(N, M=None, k=0, dtype=float32, **kwargs):
    """Ones on the k-th diagonal.  The default dtype is float32 as in the reference (ramba/ramba.py:8765-8779),
    not NumPy's float64."""
    M = N if M is None else M
    return fromfunction(lambda i, j: (i + k) == j, (N, M)).astype(dtype)


def identity(n, dtype=float32):
    return eye(n, dtype=dtype)


# =============================================================================================
# module-level functions
# =============================================================================================
HANDLED_FUNCTIONS = {}


def _as_nd(x):
    if isinstance(x, ndarray):
        return x
    if isinstance(x, np.ndarray):
        return fromarray(x)
    return x


def _unary_fn(name):
    def f(x, *args, **kwargs):
        x = _as_nd(x)
        if not isinstance(x, ndarray):
            return getattr(np, name)(x, *args, **kwargs)
        return getattr(x, name)(*args, **kwargs)

    f.__name__ = name
    HANDLED_FUNCTIONS[name] = f
    return f


# names that shadow Python builtins live in `api` and are exported by the package __init__ only
api = {}
for _n in ("abs", "square", "sqrt", "sin", "cos", "tan", "sinh", "cosh", "tanh", "arcsin", "arccos", "arctan", "exp",
           "log", "cbrt", "isfinite", "isinf", "isnan", "isneginf", "isposinf", "logical_not", "sum", "prod", "min",
           "max", "all", "any", "mean"):
    api[_n] = _unary_fn(_n)
    if _n not in ("abs", "sum", "min", "max", "all", "any"):
        globals()[_n] = api[_n]
absolute = api["abs"]
HANDLED_FUNCTIONS["absolute"] = absolute
amin, amax = api["min"], api["max"]


def _binary_fn(name, method, rmethod=None):
    def f(a, b, **kwargs):
        a, b = _as_nd(a), _as_nd(b)
        if isinstance(a, ndarray):
            return getattr(a, method)(b)
        if isinstance(b, ndarray):
            return getattr(b, rmethod or method)(a)
        return getattr(np, name)(a, b)

    f.__name__ = name
    HANDLED_FUNCTIONS[name] = f
    return f


minimum = _binary_fn("minimum", "minimum")
maximum = _binary_fn("maximum", "maximum")
logical_and = _binary_fn("logical_and", "logical_and")
logical_or = _binary_fn("logical_or", "logical_or")
logical_xor = _binary_fn("logical_xor", "logical_xor")
power = _binary_fn("power", "__pow__", "__rpow__")
add = _binary_fn("add", "__add__", "__radd__")
subtract = _binary_fn("subtract", "__sub__", "__rsub__")
multiply = _binary_fn("multiply", "__mul__", "__rmul__")
divide = _binary_fn("divide", "__truediv__", "__rtruediv__")
true_divide = divide
floor_divide = _binary_fn("floor_divide", "__floordiv__", "__rfloordiv__")
mod = _binary_fn("mod", "__mod__", "__rmod__")


def isclose(a, b, rtol=1e-5, atol=1e-8, equal_nan=False):
    """ramba.internal_isclose (ramba/ramba.py:7834-7839) spelled with fused ops."""
    a = _as_nd(a)
    b = _as_nd(b)
    if not isinstance(a, ndarray):
        a, b = b, a
        diff = absolute(b - a) if isinstance(b, ndarray) else absolute(a - b)
    else:
        diff = absolute(a - b)
    bb = absolute(b) if isinstance(b, ndarray) else builtins.abs(b)
    tol = bb * rtol + atol
    res = logical_and(isfinite(a), diff <= tol)  # noqa: F821
    res = logical_or(res, logical_and(isinf(a), a == b))  # noqa: F821
    if equal_nan:
        nb = isnan(b) if isinstance(b, ndarray) else bool(np.isnan(b))  # noqa: F821
        res = logical_or(res, logical_and(isnan(a), nb))  # noqa: F821
    return res


def allclose(a, b, rtol=1e-5, atol=1e-8, equal_nan=False):
    return bool(isclose(a, b, rtol=rtol, atol=atol, equal_nan=equal_nan).all())


def where(cond, a=None, b=None):
    """`a if cond else b` as one fused statement (ramba/ramba.py:9755-9799); with the condition alone, nonzero(cond)."""
    if a is None and b is None:
        return compaction.nonzero(cond)
    cond, a, b = _as_nd(cond), _as_nd(a), _as_nd(b)
    shape = cond.shape
    for x in (a, b):
        if isinstance(x, ndarray):
            shape = tuple(np.broadcast_shapes(shape, x.shape))

    def view(x):
        if isinstance(x, ndarray) and x.shape != () and x.shape != shape:
            return x.broadcast_to(shape)
        return x

    adt = a.dtype if isinstance(a, ndarray) else np.asarray(a).dtype
    new = empty(shape, dtype=adt)
    DAG.assign(new, E("where", view(cond), view(a), view(b)))
    return new


def clip(a, a_min, a_max, out=None):
    return a.clip(a_min, a_max, out=out)


def transpose(a, *args):
    return a.transpose(*args)


def swapaxes(a, a1, a2):
    return a.swapaxes(a1, a2)


def moveaxis(a, s, d):
    return a.moveaxis(s, d)


def broadcast_to(a, shape):
    return a.broadcast_to(shape)


def expand_dims(a, axis):
    return _as_nd(a).expand_dims(axis)


def squeeze(a, axis=None):
    return _as_nd(a).squeeze(axis)


def reshape(a, *shape):
    return _as_nd(a).reshape(*shape)


def _norm_newshape(arr, newshape):
    if isinstance(newshape, numbers.Integral):
        newshape = (newshape,)
    newshape = tuple(int(x) for x in newshape)
    if builtins.any(x < -1 for x in newshape):
        raise ValueError("Illegal dimension size in reshape.")
    total = arr.size
    if newshape.count(-1) > 1:
        raise ValueError("Too many -1 dimensions given to reshape.")
    if -1 in newshape:
        rest = int(np.prod([x for x in newshape if x != -1], dtype=np.int64))
        if rest == 0 or total % rest != 0:
            raise ValueError("Incompatible shape given to reshape.")
        newshape = tuple(total // rest if x == -1 else x for x in newshape)
    if int(np.prod(newshape, dtype=np.int64)) != total:
        raise ValueError("cannot reshape array of size %d into shape %s" % (total, newshape))
    return newshape


def reshape_copy(arr, newshape):
    """A new array of shape `newshape` holding arr's elements in C order (ramba/ramba.py:9241-9277; worker side
    RemoteState.reshape 2409-2499 moves one element at a time in Python).  Here: the blocks of both arrays are cut into
    runs of consecutive linear indices, every (source rank, destination rank) pair exchanges the intersections of its runs
    - packed into one buffer per peer, one grouped send / receive - and runs of equal length at constant steps are single
    2-D strided copies on the GPU (ramba_b200/redistribute.py)."""
    from . import redistribute as R

    arr = _as_nd(arr)
    newshape = _norm_newshape(arr, newshape)
    if arr.shape == ():
        return full(newshape, arr.distribution.item(), dtype=arr.dtype)
    # the source as a whole array in its own buffer (views, masks and padded blocks are materialised by one fused copy)
    src = arr
    if arr.base is not None or arr.maskarray is not None or arr.local_border or \
            not (arr.distribution is arr.bdarray.distribution or shardview.dist_is_eq(arr.distribution, arr.bdarray.distribution)):
        src = copy(arr)
    out = ndarray(newshape, dtype=arr.dtype, flex_dist=False)
    DAG.instantiate(src)
    W, w = common.num_workers, common.worker_num
    sdist, ddist = src.bdarray.distribution, out.bdarray.distribution
    sh_src, sh_dst = blocks.block(src), blocks.block(out)
    if arr.size == 0:
        return out
    code = rb_dtype(arr.dtype)
    isz = blocks.itemsize(arr.dtype)
    prog = _pack_program(code, code)

    def runs(shape, dist, r, shard):
        sv = dist[r]
        if shardview.is_empty(sv):
            return np.zeros(0, dtype=np.int64), 0, None
        st, ln, m = R.block_runs(shape, sv.start, sv.size, True)
        loc = None
        if shard is not None:
            loc = R.run_local_offsets(sv.size, m, shard.strides, 0)
        return st, ln, loc

    my_s, my_sl, my_sloc = runs(src.shape, sdist, w, sh_src)
    my_d, my_dl, my_dloc = runs(out.shape, ddist, w, sh_dst)

    def copy_groups(length, so, do, sptr, dptr, sbounds, dbounds):
        for (i0, cnt, ln, ds, dd) in R.strided_groups(length, so, do):
            a = (sptr + int(so[i0]) * isz, [ds, 1], code) + ((sbounds,) if sbounds is not None else ())
            b = (dptr + int(do[i0]) * isz, [dd, 1], code) + ((dbounds,) if dbounds is not None else ())
            RT.launch(prog, [cnt, ln], [0, 0], [a, b])

    # pieces that stay on this rank
    ia, ib, ps, pl = R.intersect_runs(my_s, my_sl, my_d, my_dl)
    if len(ps):
        copy_groups(pl, my_sloc[ia] + (ps - my_s[ia]), my_dloc[ib] + (ps - my_d[ib]), sh_src.ptr(0), sh_dst.ptr(0), sh_src.bounds, sh_dst.bounds)
    if W == 1:
        return out
    ops, unpack = [], []
    tdt = torch_dtype(arr.dtype)
    for peer in range(W):
        if peer == w:
            continue
        # what `peer` needs from my source block, in linear order
        p_d, p_dl, _ = runs(out.shape, ddist, peer, None)
        ia, ib, ps, pl = R.intersect_runs(my_s, my_sl, p_d, p_dl)
        if len(ps):
            n = int(pl.sum())
            buf = torch.empty(n, dtype=tdt, device=RT.device)
            copy_groups(pl, my_sloc[ia] + (ps - my_s[ia]), np.cumsum(pl) - pl, sh_src.ptr(0), buf.data_ptr(), sh_src.bounds, None)
            ops.append((True, buf, peer))
        # what I need from `peer`'s source block
        p_s, p_sl, _ = runs(src.shape, sdist, peer, None)
        ia, ib, ps, pl = R.intersect_runs(p_s, p_sl, my_d, my_dl)
        if len(ps):
            n = int(pl.sum())
            buf = torch.empty(n, dtype=tdt, device=RT.device)
            ops.append((False, buf, peer))
            unpack.append((pl, np.cumsum(pl) - pl, my_dloc[ib] + (ps - my_d[ib]), buf))
    for wk in RT.p2p(ops):
        wk.wait()  # (the launching stream waits; the host does not)
    for (pl, so, do, buf) in unpack:
        copy_groups(pl, so, do, buf.data_ptr(), sh_dst.ptr(0), None, sh_dst.bounds)
    RT.hold(*[b for (_, b, _) in ops])
    return out


def ndim(a):
    return a.ndim if hasattr(a, "ndim") else np.ndim(a)


def result_type(*args):
    return np.result_type(*[a.dtype if isinstance(a, ndarray) else a for a in args])


def isscalar(x):
    return np.isscalar(x)


for _n in ("where", "clip", "transpose", "swapaxes", "moveaxis", "broadcast_to", "expand_dims", "squeeze", "reshape", "ndim", "result_type", "allclose",
           "isclose", "empty_like", "zeros_like", "ones_like", "full_like", "copy", "array"):
    HANDLED_FUNCTIONS[_n] = globals()[_n]


# ---- stencil skeleton (ramba/ramba.py:441-541, 9987-10054) ---------------------------------------
class StencilMetadata:
    """`@stencil` function with relative indexing (`a[-1, 0] + a[1, 0]`).  The reference compiles it
    with numba.stencil; here it is evaluated symbolically: every relative access becomes a shifted
    slice view of the interior, so the whole stencil is one fused op on the N-d kernel."""

    def __init__(self, func):
        self.func = func
        self.neighborhood = None

    def __call__(self, *args, **kwargs):
        return sstencil(self, *args, **kwargs)


def stencil(*args, **kwargs):
    if len(args) == 1 and callable(args[0]) and not kwargs:
        return StencilMetadata(args[0])

    def rdec(func):
        return StencilMetadata(func)

    return rdec


class _RelRecorder:
    """First pass: records the relative offsets a stencil function touches."""

    def __init__(self, ndim, offsets):
        self.ndim, self.offsets = ndim, offsets

    def __getitem__(self, idx):
        idx = idx if isinstance(idx, tuple) else (idx,)
        if len(idx) != self.ndim or not builtins.all(isinstance(i, numbers.Integral) for i in idx):
            raise IndexError("stencil functions index their array arguments with one constant relative offset per dimension")
        self.offsets.append(tuple(int(i) for i in idx))
        return 1.0


class _RelView:
    """Second pass: a relative access is the interior box shifted by the offset."""

    def __init__(self, arr, lo, hi):
        self.arr, self.lo, self.hi = arr, lo, hi

    def __getitem__(self, idx):
        idx = idx if isinstance(idx, tuple) else (idx,)
        sl = tuple(slice(-self.lo[d] + idx[d], self.arr.shape[d] - self.hi[d] + idx[d]) for d in range(len(idx)))
        return self.arr[sl]


def sstencil(func, *args, out=None, **kwargs):
    """Apply a `@stencil` function to distributed arrays: interior = stencil expression, border = 0
    (numba.stencil's cval) or left untouched when `out` is given."""
    if not isinstance(func, StencilMetadata):
        func = StencilMetadata(func)
    arrays = [a for a in args if isinstance(a, ndarray)]
    assert len(arrays) > 0, "sstencil needs at least one distributed array argument"
    shape = arrays[0].shape
    for a in arrays:
        assert a.shape == shape, "sstencil: array arguments must have the same shape"
    k = len(shape)
    if func.neighborhood is None:
        offs = []
        func.func(*[_RelRecorder(k, offs) if isinstance(a, ndarray) else a for a in args])
        lo = tuple(builtins.min([0] + [o[d] for o in offs]) for d in range(k))
        hi = tuple(builtins.max([0] + [o[d] for o in offs]) for d in range(k))
        func.neighborhood = tuple((lo[d], hi[d]) for d in range(k))
    lo = tuple(n[0] for n in func.neighborhood)
    hi = tuple(n[1] for n in func.neighborhood)
    res = func.func(*[_RelView(a, lo, hi) if isinstance(a, ndarray) else a for a in args])
    if out is not None:
        new = out
    elif arrays[0].local_border > 0:
        # like the reference: allocated with the divisions and the border of the first argument (ramba/ramba.py:10022-10026)
        new = create_array_with_divisions(shape, arrays[0].distribution, local_border=arrays[0].local_border,
                                          dtype=res.dtype if isinstance(res, ndarray) else np.float64)
        DAG.assign(new, 0)
    else:
        new = zeros(shape, dtype=res.dtype if isinstance(res, ndarray) else np.float64)
    interior = tuple(slice(-lo[d], shape[d] - hi[d]) for d in range(k))
    new[interior] = res
    return new


# =============================================================================================
# joining and padding: concatenate / stack / pad.  The reference has dedicated redistribution executors
# (ramba/ramba.py:9479-9590, 9280-9420); here the result is allocated with the default distribution and filled by
# ordinary slice assignments, i.e. fused copy ops whose source pieces cross ranks through the generic piece
# exchange of run_deferred_ops.
# =============================================================================================
def concatenate(arrayseq, axis=0, out=None, **kwargs):
    assert out is None, "concatenate(out=...) is not supported"
    arrays = [_as_nd(a) for a in arrayseq]
    assert len(arrays) > 0 and builtins.any(isinstance(a, ndarray) for a in arrays)
    first = arrays[0]
    axis = axis % first.ndim
    out_shape = list(first.shape)
    for a in arrays[1:]:
        assert a.ndim == first.ndim, "all the input arrays must have the same number of dimensions"
        assert a.dtype == first.dtype, "concatenate: dtypes must match (ramba/ramba.py:9566)"
        for i in range(first.ndim):
            if i == axis:
                out_shape[i] += a.shape[i]
            else:
                assert a.shape[i] == first.shape[i], "all the input array dimensions except for the concatenation axis must match"
    res = empty(tuple(out_shape), dtype=first.dtype)
    at = 0
    for a in arrays:
        sl = tuple(slice(at, at + a.shape[i]) if i == axis else slice(None) for i in range(first.ndim))
        if a.shape[axis] > 0:
            res[sl] = a
        at += a.shape[axis]
    return res


def stack(arrays, axis=0, out=None):
    assert out is None, "stack(out=...) is not supported"
    arrays = [_as_nd(a) for a in arrays]
    assert builtins.all(a.shape == arrays[0].shape for a in arrays), "all input arrays must have the same shape"
    axis = axis % (arrays[0].ndim + 1)
    return concatenate([a.expand_dims(axis) for a in arrays], axis=axis)


def pad(arr, pad_width, mode="constant", **kwargs):
    """NumPy's pad for the modes the reference has: constant (with constant_values), edge, wrap, empty
    (ramba/ramba.py:9400-9420).  Axes are padded one after the other, like NumPy does, so corners come out right."""
    arr = _as_nd(arr)
    assert arr.ndim >= 1
    assert mode in ("constant", "empty", "edge", "wrap")
    if isinstance(pad_width, numbers.Integral):
        pad_width = (pad_width, pad_width)
    if not isinstance(pad_width[0], (tuple, list)):
        pad_width = tuple(tuple(pad_width) if len(pad_width) == 2 else (pad_width[0], pad_width[0]) for _ in range(arr.ndim))
    assert arr.ndim == len(pad_width)
    cvals = kwargs.get("constant_values", 0)
    if isinstance(cvals, numbers.Number):
        cvals = ((cvals, cvals),) * arr.ndim
    elif not isinstance(cvals[0], (tuple, list)):
        cvals = (tuple(cvals),) * arr.ndim
    elif len(cvals) == 1:
        cvals = tuple(cvals) * arr.ndim
    cur = arr
    for ax in range(arr.ndim):
        before, after = int(pad_width[ax][0]), int(pad_width[ax][1])
        if before == 0 and after == 0:
            continue
        n = cur.shape[ax]
        shape = tuple(cur.shape[i] + (before + after if i == ax else 0) for i in range(cur.ndim))

        def region(lo, hi):
            return tuple(slice(lo, hi) if i == ax else slice(None) for i in range(cur.ndim))

        new = empty(shape, dtype=cur.dtype)
        new[region(before, before + n)] = cur
        if mode == "constant":
            if before:
                new[region(0, before)] = cvals[ax][0]
            if after:
                new[region(before + n, before + n + after)] = cvals[ax][1]
        elif mode == "edge":
            if before:
                new[region(0, before)] = cur[region(0, 1)]
            if after:
                new[region(before + n, before + n + after)] = cur[region(n - 1, n)]
        elif mode == "wrap":
            assert before <= n and after <= n, "pad(mode='wrap') wider than the array is not supported"
            if before:
                new[region(0, before)] = cur[region(n - before, n)]
            if after:
                new[region(before + n, before + n + after)] = cur[region(0, after)]
        cur = new
    return cur if cur is not arr else copy(arr)


def split(arr, indices_or_sections, axis=0):
    """Equal sections (like the reference, ramba/ramba.py:9593-9611) or NumPy's list of split points, as views."""
    arr = _as_nd(arr)
    axis = axis % arr.ndim
    n = arr.shape[axis]
    if isinstance(indices_or_sections, numbers.Integral):
        if n % indices_or_sections != 0:
            raise ValueError(f"Cannot evenly divide array dimension of length {n} into {indices_or_sections} equal sections.")
        step = n // indices_or_sections
        bounds = [(k * step, (k + 1) * step) for k in range(indices_or_sections)]
    else:
        pts = [0] + [builtins.min(int(p), n) for p in indices_or_sections] + [n]
        bounds = [(pts[k], builtins.max(pts[k], pts[k + 1])) for k in range(len(pts) - 1)]
    return [arr[tuple(slice(lo, hi) if d == axis else slice(None) for d in range(arr.ndim))] for lo, hi in bounds]


def rollaxis(a, axis, start=0):
    return _as_nd(a).rollaxis(axis, start)


def nansum(a, **kwargs):
    return _as_nd(a).nansum(**kwargs)


def nanmean(a, axis=None, dtype=None):
    return _as_nd(a).nanmean(axis=axis, dtype=dtype)


for _n in ("concatenate", "stack", "pad", "split", "rollaxis", "nansum", "nanmean"):
    HANDLED_FUNCTIONS[_n] = globals()[_n]


# ---- first-occurrence index reductions on the index-reduction kernel (ramba_b200/argreduce.py)
def argmax(a, axis=None, out=None, *, keepdims=False):
    return argreduce.arg_reduce(a, "argmax", axis, out, keepdims)


def argmin(a, axis=None, out=None, *, keepdims=False):
    return argreduce.arg_reduce(a, "argmin", axis, out, keepdims)


def nanargmax(a, axis=None, out=None, *, keepdims=False):
    return argreduce.arg_reduce(a, "nanargmax", axis, out, keepdims)


def nanargmin(a, axis=None, out=None, *, keepdims=False):
    return argreduce.arg_reduce(a, "nanargmin", axis, out, keepdims)


ndarray.argmax = argmax
ndarray.argmin = argmin
for _n in ("argmax", "argmin", "nanargmax", "nanargmin"):
    HANDLED_FUNCTIONS[_n] = globals()[_n]


# ---- stream compaction on the compaction kernel (ramba_b200/compaction.py)
nonzero = compaction.nonzero
flatnonzero = compaction.flatnonzero
argwhere = compaction.argwhere
count_nonzero = compaction.count_nonzero
extract = compaction.extract


def compress(condition, a, axis=None, out=None):
    if out is not None:
        raise NotImplementedError("compress: out= is not supported")
    return compaction.compress(condition, a, axis)


ndarray.nonzero = nonzero
ndarray.compress = lambda self, condition, axis=None, out=None: compress(condition, self, axis, out)
for _n in ("nonzero", "flatnonzero", "argwhere", "count_nonzero", "extract", "compress"):
    HANDLED_FUNCTIONS[_n] = globals()[_n]


# ---- binning on the histogram and bin-search kernels (ramba_b200/binning.py)
histogram = binning.histogram
histogram_bin_edges = binning.histogram_bin_edges
bincount = binning.bincount
searchsorted = binning.searchsorted
digitize = binning.digitize
ndarray.searchsorted = lambda self, v, side="left", sorter=None: searchsorted(self, v, side, sorter)
for _n in ("histogram", "histogram_bin_edges", "bincount", "searchsorted", "digitize"):
    HANDLED_FUNCTIONS[_n] = globals()[_n]


# ---- order statistics on the radix-select kernels (ramba_b200/quantile.py)
median = _quantile_mod.median
nanmedian = _quantile_mod.nanmedian
percentile = _quantile_mod.percentile
nanpercentile = _quantile_mod.nanpercentile
quantile = _quantile_mod.quantile
nanquantile = _quantile_mod.nanquantile
for _n in ("median", "nanmedian", "percentile", "nanpercentile", "quantile", "nanquantile"):
    HANDLED_FUNCTIONS[_n] = globals()[_n]


# =============================================================================================
# index-driven builders: triu / tril / select / mgrid / meshgrid.  The reference runs a per-worker NumPy
# routine for each (ramba/ramba.py:2091-2111 triu, 8993-9050 mgrid/meshgrid, 9079-9092 select); here they are
# ordinary fused elementwise ops over iota operands.
# =============================================================================================
def triu(m, k=0):
    """Upper triangle of a 2-D array: elements below the k-th diagonal zeroed (ramba/ramba.py:9053-9076)."""
    m = _as_nd(m)
    assert m.ndim == 2, "triu needs a 2-D array"
    i, j = _index_arrays(m.shape)
    return where(j - i >= k, m, zeros(m.shape, dtype=m.dtype))


def tril(m, k=0):
    """Lower triangle of a 2-D array (NumPy's tril; the reference has only triu)."""
    m = _as_nd(m)
    assert m.ndim == 2, "tril needs a 2-D array"
    i, j = _index_arrays(m.shape)
    return where(j - i <= k, m, zeros(m.shape, dtype=m.dtype))


def select(condlist, choicelist, default=0):
    """The reference's select (ramba/ramba.py:9079-9092), reproduced as written: a float64 array filled with
    `default`, then masked assignments in the order condlist[0], condlist[-1], condlist[-2], ... (its loop
    indexes with -i), so where several conditions hold the one applied LAST wins - not NumPy's first-match
    rule."""
    assert len(condlist) == len(choicelist) and len(condlist) > 0
    shape = condlist[0].shape
    for c in list(condlist) + [x for x in choicelist if isinstance(x, ndarray)]:
        assert c.shape == shape
    temp = full(shape, default)
    for i in range(len(choicelist)):
        temp[condlist[-i]] = choicelist[-i]
    return temp


def _stack_by_first_index(parts, shape, dtype):
    """Array of shape (len(parts),) + shape whose slab d is parts[d](index arrays of the trailing dims)."""
    idx = _index_arrays((len(parts),) + tuple(shape))
    out = parts[-1](idx[1:])
    if not isinstance(out, ndarray):
        out = full((len(parts),) + tuple(shape), out, dtype=dtype)
    for d in range(len(parts) - 2, -1, -1):
        out = where(idx[0] == d, parts[d](idx[1:]), out)
    return out if out.dtype == np.dtype(dtype) else out.astype(dtype)


class MgridGen:
    """`mgrid[a0:b0, a1:b1, ...]` -> int64 array of shape (k, b0-a0, b1-a1, ...) (ramba/ramba.py:9001-9018:
    unit steps only)."""

    def __getitem__(self, index):
        if isinstance(index, slice):  # NumPy: a bare slice gives the 1-D grid itself
            assert index.step is None, "mgrid supports unit-step slices"
            return arange(0 if index.start is None else int(index.start), int(index.stop))
        index = index if isinstance(index, tuple) else (index,)
        starts, sizes = [], []
        for ix in index:
            if isinstance(ix, numbers.Integral):
                starts.append(0)
                sizes.append(int(ix))
            else:
                assert isinstance(ix, slice) and ix.step is None, "mgrid supports unit-step slices"
                starts.append(0 if ix.start is None else int(ix.start))
                sizes.append(int(ix.stop) - starts[-1])
        parts = [(lambda tail, d=d: tail[d] + starts[d]) for d in range(len(index))]
        return _stack_by_first_index(parts, sizes, np.int64)


mgrid = MgridGen()


def meshgrid(*xi, copy=True, sparse=False, indexing="xy"):
    """`meshgrid(x0, x1, ..., indexing='ij')` of equal-dtype 1-D arrays as ONE array of shape (k, n0, n1, ...)
    (the reference's restrictions, ramba/ramba.py:9028-9050)."""
    if indexing != "ij":
        raise ValueError("Unsupported meshgrid indexing option %s" % (indexing,))
    if sparse is not False:
        raise ValueError("Unsupported meshgrid sparse option %s" % (sparse,))
    if copy is not True:
        raise ValueError("Unsupported meshgrid copy option %s" % (copy,))
    xs = [_as_nd(x) if isinstance(x, (ndarray, np.ndarray)) else x for x in xi]
    if builtins.any(not (isinstance(x, ndarray) and x.ndim == 1) for x in xs):
        raise ValueError("Unsupported argument to meshgrid")
    if not builtins.all(x.dtype == xs[0].dtype for x in xs):
        raise ValueError("Mis-matching dtypes to meshgrid")
    k = len(xs)
    sizes = [x.shape[0] for x in xs]
    full_shape = (k,) + tuple(sizes)

    def part(d):
        # x_d varies along axis d+1 of the result and is broadcast along the others
        def f(tail):
            others = [sizes[e] for e in range(k) if e != d]
            b = broadcast_to(xs[d], (k,) + tuple(others) + (sizes[d],))  # x_d along the last axis ...
            return moveaxis(b, -1, d + 1)  # ... moved to its own axis
        return f

    return _stack_by_first_index([part(d) for d in range(k)], sizes, xs[0].dtype)


# =============================================================================================
# skeletons over user functions: smap / smap_index / sreduce / sreduce_index / cumsum
# (ramba/ramba.py:9863-9984, 9675-9679, 10057-10116).  The reference pickles the function to its workers and
# lets Numba compile it per element; here the function is evaluated ONCE on lazy arrays and lands in the same
# fused op list as every other expression, so it has to be built from array operators and ramba functions
# (no data-dependent Python control flow; `where` is the select).
# =============================================================================================
def _user_function(func):
    """A callable, or a string holding a lambda (the reference's string form, ramba/ramba.py:9877-9891)."""
    if isinstance(func, str):
        import sys

        mod = sys.modules[__name__.rsplit(".", 1)[0]]  # the package: numpy-like namespace for the lambda's globals
        return eval(func, {"numpy": mod, "np": mod, "ramba": mod, "math": mod})
    if not callable(func):
        raise TypeError("expected a function or a string holding a lambda")
    return func


def _first_array(args, what):
    arrays = [a for a in args if isinstance(a, ndarray)]
    assert len(arrays) > 0, what + " needs at least one distributed array argument"
    for a in arrays:
        assert a.shape == arrays[0].shape, what + ": array arguments must have the same shape"
    return arrays[0]


def _index_arrays(shape):
    idx = []
    for d in range(len(shape)):
        a = empty(shape, dtype=np.int64)
        DAG.assign(a, Iota(d))
        idx.append(a)
    return idx


_KEEP_DTYPE = object()  # sreduce: keep the mapped values in the function's own result dtype


def _smap(what, func, args, dtype, axis, with_index):
    if axis is not None:
        raise NotImplementedError(what + "(axis=...) (slice-wise functions) is not supported by the op-list backend")
    f = _user_function(func)
    first = _first_array(args, what)
    if with_index:
        idx = _index_arrays(first.shape)
        # 1-D: the index is a scalar, N-d: a tuple (ramba/ramba.py:9881-9885)
        res = f(idx[0] if first.ndim == 1 else tuple(idx), *args)
    else:
        res = f(*args)
    if not isinstance(res, ndarray):
        res = _full_of(first.shape, res)
    # the output has the dtype of the first array argument unless told otherwise (ramba/ramba.py:9872-9873, 9913-9914)
    if res.shape != first.shape:
        res = broadcast_to(res, first.shape) + zeros(first.shape, dtype=res.dtype)
    if dtype is _KEEP_DTYPE:
        return res
    out_dtype = np.dtype(first.dtype if dtype is None else dtype)
    return res if res.dtype == out_dtype else res.astype(out_dtype)


def smap(func, *args, dtype=None, parallel=True, axis=None, imports=[]):
    """Elementwise map of `func` over the array arguments (scalars pass through)."""
    return _smap("smap", func, args, dtype, axis, False)


def smap_index(func, *args, dtype=None, parallel=True, imports=[]):
    """Like smap; `func` receives the global index first (a scalar for 1-D arrays, a tuple otherwise)."""
    return _smap("smap_index", func, args, dtype, None, True)


class SreduceReducer:
    """(worker function, driver function) pair of the reference's sreduce (ramba/ramba.py:9934-9939)."""

    __slots__ = ("worker_func", "driver_func")

    def __init__(self, worker_func, driver_func):
        self.worker_func = worker_func
        self.driver_func = driver_func


def _classify_reducer(reducer):
    """The op-list backend reduces with +, *, min or max: recognise which one `reducer` is by probing it."""
    probes = [(3, 5), (-2, 7), (4, 4), (0.5, -8.0)]
    table = {"sum": lambda a, b: a + b, "prod": lambda a, b: a * b, "min": builtins.min, "max": builtins.max}
    for name, ref in table.items():
        try:
            if builtins.all(reducer(a, b) == ref(a, b) for a, b in probes):
                return name
        except Exception:
            pass
    raise NotImplementedError("sreduce: the reducer must be +, *, min or max (element-by-element Python reducers cannot run on the GPU)")


def _sreduce(what, func, reducer, identity, args, with_index):
    if isinstance(reducer, SreduceReducer):
        reducer = reducer.worker_func
    red = _user_function(reducer)
    kind = _classify_reducer(red)
    mapped = _smap(what, func, args, _KEEP_DTYPE, None, with_index)
    total = getattr(mapped, kind)()
    if isinstance(total, ndarray):
        total = total.asarray().reshape(-1)[0]
    return red(identity, total)


def sreduce(func, reducer, identity, *args, parallel=True):
    """reduce(reducer, map(func, elements), identity) (ramba/ramba.py:9942-9980)."""
    return _sreduce("sreduce", func, reducer, identity, args, False)


def sreduce_index(func, reducer, identity, *args, parallel=True):
    return _sreduce("sreduce_index", func, reducer, identity, args, True)


def _scan_native(a, axis, kind, dtype):
    """cumsum / cumprod / running min / max along `axis` with the single-pass scan kernel (rb200_cumulative): every
    rank scans its own block; when the array is cut along the scan axis the block totals are all-gathered and every rank
    folds the totals of the blocks before its own into its part (the reference passes boundary values worker to worker,
    ramba/ramba.py:3378-3437).  Returns None when this layout / dtype is not covered (caller falls back)."""
    out_dtype = np.dtype(dtype) if dtype is not None else a.dtype
    if out_dtype.kind in "iub" and out_dtype.itemsize < 8:
        out_dtype = np.dtype(np.int64)  # NumPy: small integers accumulate in the platform integer
    if out_dtype not in (np.dtype(np.float64), np.dtype(np.float32), np.dtype(np.int64)):
        return None
    W, w = common.num_workers, common.worker_num
    # a whole array in the result dtype, in its own buffer: views / other dtypes are materialised by one fused copy
    src = a.astype(out_dtype) if (a.dtype != out_dtype or a.base is not None or a.maskarray is not None) else a
    DAG.instantiate(src)
    dist = src.bdarray.distribution
    if src.base is not None or src.distribution is not dist and not shardview.dist_is_eq(src.distribution, dist):
        return None
    nd = src.ndim
    split_axis = builtins.any(not shardview.is_empty(sv) and (int(sv.start[axis]) != 0 or int(sv.size[axis]) != src.shape[axis]) for sv in dist)
    if split_axis:
        for sv in dist:  # cut along the scan axis ONLY: every rank's totals cover the same columns
            if shardview.is_empty(sv):
                continue
            if builtins.any(int(sv.start[d]) != 0 or int(sv.size[d]) != src.shape[d] for d in range(nd) if d != axis):
                return None
    res = create_array_with_divisions(src.shape, dist, dtype=out_dtype)
    sh_src, sh_res = blocks.block(src), blocks.block(res)
    if sh_src.border:
        return None
    lshape = sh_src.shape
    mine_empty = shardview.is_empty(dist[w])
    n_outer = int(np.prod(lshape[:axis])) if not mine_empty else 0
    length = int(lshape[axis]) if not mine_empty else 0
    n_inner = int(np.prod(lshape[axis + 1:])) if not mine_empty else 1
    code = rb_dtype(out_dtype)
    red = REDUCTIONS[kind]
    acc_dt = torch.float64 if out_dtype.kind == "f" else torch.int64
    ncols = int(np.prod([src.shape[d] for d in range(nd) if d != axis]))
    totals = torch.empty(max(1, ncols), dtype=acc_dt, device=RT.device) if split_axis else None
    if totals is not None:
        totals.fill_(red.identity(out_dtype))
    scratch = carry = rescan = None
    if not mine_empty:
        scratch = RT.cumulative(sh_src.ptr(0), sh_res.ptr(0), code, n_outer, length, n_inner, red.code, None, totals.data_ptr() if totals is not None else None)
    if split_axis and W > 1:
        allt = torch.empty(W * ncols, dtype=acc_dt, device=RT.device)
        RT.all_gather(allt, totals).wait()
        if not mine_empty:
            before = [p for p in range(W) if not shardview.is_empty(dist[p]) and int(dist[p].start[axis]) < int(dist[w].start[axis])]
            if before:
                stack = allt.view(W, ncols)[before]
                carry = red.fold(stack).contiguous()
                # scan the block again seeded with the carry, so that the carry joins the float64 accumulator and every
                # element is rounded once, as at one rank (folding the carry into the stored result would round twice)
                rescan = RT.cumulative(sh_src.ptr(0), sh_res.ptr(0), code, n_outer, length, n_inner, red.code, carry.data_ptr(), None)
    RT.hold(scratch, carry, rescan)  # (read only by the launches above)
    return res


def scumulative(local_func, final_func, array, axis=None, dtype=None, out=None):
    """Inclusive scan with a user function (ramba/ramba.py:10057-10116): the reference scans every worker's part with
    `local_func` and then folds the boundary values in with `final_func`.  When `local_func` is +, *, min or max
    (recognised by probing, like sreduce) the single-pass scan kernel runs it; any other traceable associative
    function is applied in log2(n) shifted-slice steps on the elementwise kernels."""
    array = _as_nd(array)
    if array.ndim == 1 and axis is None:
        axis = 0
    assert isinstance(axis, numbers.Number) and 0 <= axis < array.ndim, "scumulative needs an axis for N-d arrays"
    assert out is None, "scumulative(out=...) is not supported (nor by the reference, ramba/ramba.py:10071-10075)"
    f = _user_function(local_func)
    try:
        kind = _classify_reducer(f)
    except NotImplementedError:
        kind = None
    return _scan(array, int(axis), kind, f, dtype)


def _scan(a, axis, kind, step, dtype):
    """Inclusive scan of `a` along `axis`: reduction `kind` on the scan kernel when it covers the layout, otherwise (or
    when kind is None) log2(n) fused shifted-slice steps `hi = step(lo, hi)`."""
    if kind is not None and a.size > 0:
        res = _scan_native(a, axis, kind, dtype)
        if res is not None:
            return res
    cur = a.astype(dtype) if dtype is not None and np.dtype(dtype) != a.dtype else a + 0
    n = a.shape[axis]
    d = 1
    while d < n:
        nxt = cur + 0  # fresh array: a step reads the previous one at two offsets, it cannot run in place
        hi = tuple(slice(d, None) if k == axis else slice(None) for k in range(a.ndim))
        lo = tuple(slice(0, n - d) if k == axis else slice(None) for k in range(a.ndim))
        nxt[hi] = step(cur[lo], cur[hi])
        cur = nxt
        d *= 2
    return cur


def cumsum(a, axis=None, dtype=None, out=None):
    """Cumulative sum along `axis` (ramba/ramba.py:9675-9679).  The reference scans each worker's part and then adds the
    boundary values worker by worker; here every rank's block is scanned in ONE pass over HBM by the decoupled-look-back
    scan kernel (rb200_cumulative) and, when the array is cut along the axis, the block totals travel by one all-gather.
    Integer and exactly representable data agree with NumPy bit for bit; floating-point sums are associated differently
    (as they are in the reference).  Layouts the kernel does not cover (2-D block partitions cut along and across the
    axis) fall back to log2(n) fused shifted-slice additions."""
    a = _as_nd(a)
    if a.ndim == 1 and axis is None:
        axis = 0
    assert isinstance(axis, numbers.Number) and 0 <= axis < a.ndim, "cumsum needs an axis for N-d arrays"
    assert out is None, "cumsum(out=...) is not supported (nor by the reference, ramba/ramba.py:10071-10075)"
    return _scan(a, int(axis), "sum", lambda lo, hi: hi + lo, dtype)


def instantiate_all(*args, **kwargs):
    """Make sure all arrays among the arguments have been computed (ramba/ramba.py:5318-5324)."""
    for a in args:
        if isinstance(a, ndarray):
            a.instantiate()


def sync():
    """Flush pending fused ops and wait for this rank's GPU (ramba/ramba.py:9843-9849)."""
    t0 = timer()
    DAG.execute_all()
    deferred_op.do_ops()
    RT.synchronize()
    add_time("sync", timer() - t0)


def timing_summary():
    """Per-phase wall-clock totals (RAMBA_TIMING, ramba/ramba.py:954-997, 7620-7627)."""
    txt = common.get_timing_str(details=True)
    if txt:
        print("ramba_b200 timing (rank %d):\n%s\nlaunches: %d, bytes sent to peers: %d" % (common.worker_num, txt, RT.launches, RT.bytes_sent))
        print("DAG: %d statements deferred, %d executed, %d never needed, %d pending; memos: %d lowerings, %d flush plans / scripts"
              % (DAG.dag_count, DAG.executed_count, DAG.pruned_count, len(DAG.pending), len(_lower_cache), len(_plan_cache)))


def print_comm_stats():
    print("ramba_b200 rank %d: %d bytes sent to peers, %d kernel launches" % (common.worker_num, RT.bytes_sent, RT.launches))


if common.ntiming > 0:
    import atexit

    atexit.register(timing_summary)


def get_timing(details=False):
    return common.get_timing(details)


def get_timing_str(details=False):
    return common.get_timing_str(details)


def reset_timing():
    common.reset_timing()
