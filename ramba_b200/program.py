"""Fused-op IR and its lowering to the op-list accumulator machine of libramba_b200.

The reference's fuser accumulates *Python source lines* (`tmp_k = f(tmp_i, tmp_j)`), substitutes
`[index]` for live arrays and lets Numba type and compile the loop body
(ramba/ramba.py:8198-8265).  Here the same statements are expression trees; this module

  * types them the way Numba types the reference's scalar loop body (array elements keep their
    dtype class, Python scalars are float64/int64, ramba/ramba.py:8094-8104, 3661-3666; dead
    arrays become un-rounded scalar temporaries, ramba/ramba.py:8123-8127),
  * lowers them to instructions `acc = op(a, b[, c])` whose operands are the accumulator, a
    spill register, a view element, a scalar or an index (`index[d] + global_start[d]`,
    ramba/ramba.py:8955-8960), and
  * allocates spill registers only for values that are not consumed by the very next
    instruction.

The output (`Program`) is position independent: the same program is bound to every iteration
range of a flush (ramba/ramba.py:3758-3780 calls the same compiled function per range).
"""
import functools
import operator
import struct

import numpy as np

from . import _cabi as cabi
from ._cabi import K_ACC, K_IOTA, K_NONE, K_REG, K_SCAL, K_VIEW, NOSTORE, OP, T_F32, T_F64, T_I64

_NP2RB = {
    np.dtype(np.float64): cabi.F64,
    np.dtype(np.float32): cabi.F32,
    np.dtype(np.int64): cabi.I64,
    np.dtype(np.int32): cabi.I32,
    np.dtype(np.bool_): cabi.BOOL,
    np.dtype(np.uint8): cabi.U8,
    np.dtype(np.int8): cabi.I8,
    np.dtype(np.int16): cabi.I16,
    np.dtype(np.uint16): cabi.U16,
    np.dtype(np.uint32): cabi.U32,
}
_RB2NP = {v: k for k, v in _NP2RB.items()}


def rb_dtype(dt):
    dt = np.dtype(dt)
    if dt not in _NP2RB:
        raise TypeError("ramba_b200: dtype %s is not supported by the sm_90a fused-op kernels" % dt)
    return _NP2RB[dt]


def np_dtype(code):
    return _RB2NP[code]


def getminmax(dtype):
    dtype = np.dtype(dtype)
    if dtype.kind == "f":
        return (-np.inf, np.inf)
    if dtype.kind == "b":
        return (False, True)
    i = np.iinfo(dtype)
    return (i.min, i.max)


class Reduction:
    """What one reduction means to each part of the engine.  code: the kernel's RED_* code (stage 1, partial folds,
    the scan); combine: the E operator that folds two partials (stage 2, the scan's carry); allreduce: the
    torch.distributed ReduceOp name; identity(dtype): what an empty reduction starts from and what a masked-out element
    contributes; fold(stack): the torch fold of a stack of partials along dim 0 (the scan's carry); truth: the result
    is a truth value (all / any reduce 0/1 values, so min / max all-reduce them)."""

    __slots__ = ("code", "combine", "allreduce", "identity", "fold", "truth")

    def __init__(self, code, combine, allreduce, identity, fold, truth=False):
        self.code, self.combine, self.allreduce, self.identity, self.fold, self.truth = code, combine, allreduce, identity, fold, truth


REDUCTIONS = {
    # (the fold adds the rows in order from the first: torch's sum starts from +0.0 and would turn a -0.0 carry into +0.0)
    "sum": Reduction(cabi.RED_ADD, "add", "SUM", lambda dt: 0, lambda s: functools.reduce(operator.add, s.unbind(0))),
    "prod": Reduction(cabi.RED_MUL, "mul", "PRODUCT", lambda dt: 1, lambda s: s.prod(0)),
    "min": Reduction(cabi.RED_MIN, "min", "MIN", lambda dt: getminmax(dt)[1], lambda s: s.min(0).values),
    "max": Reduction(cabi.RED_MAX, "max", "MAX", lambda dt: getminmax(dt)[0], lambda s: s.max(0).values),
    "all": Reduction(cabi.RED_MUL, "mul", "MIN", lambda dt: 1, lambda s: s.min(0).values, truth=True),
    "any": Reduction(cabi.RED_ADD, "add", "MAX", lambda dt: 0, lambda s: s.max(0).values, truth=True),
}


def fold_expr(combine, a, b):
    """E folding partial b into partial a with a reduction's combine operator.  For min / max a NaN on either side
    wins (NumPy's reductions); the min / max binop alone is builtins.min / max, which keeps a NaN only in a."""
    e = E(combine, a, b)
    if combine in ("min", "max"):
        e = E("where", E("ne", b, b), b, e)
    return e


def red_identity(op, dtype):
    """The identity of reduction `op` (sum prod min max all any) over values of `dtype`."""
    return REDUCTIONS[op].identity(dtype)


def dtype_class(code):
    """Compute class an element of storage dtype `code` has inside the loop body."""
    if code == cabi.F64:
        return T_F64
    if code == cabi.F32:
        return T_F32
    return T_I64


def class_storage(cls):
    return {T_F64: cabi.F64, T_F32: cabi.F32, T_I64: cabi.I64}[cls]


class Iota:
    """`index[dim] + global_start[dim]` of the iteration space (int64)."""

    __slots__ = ("dim",)

    def __init__(self, dim):
        self.dim = dim


class E:
    """Expression node: op name (lower-case rb200 opcode name) + operands."""

    __slots__ = ("op", "args", "imm")

    def __init__(self, op, *args, imm=0):
        self.op = op
        self.args = args
        self.imm = imm


# ------------------------------------------------------------------------------------------
# typed operands used during lowering


class TV:
    """A typed value: compute class + bool flag + where it comes from."""

    __slots__ = ("cls", "is_bool", "kind", "ref")

    def __init__(self, cls, is_bool, kind, ref):
        self.cls = cls
        self.is_bool = is_bool
        self.kind = kind  # 'node' | 'view' | 'scal' | 'iota'
        self.ref = ref


class Node:
    __slots__ = ("op", "ctype", "rcls", "is_bool", "args", "imm", "store", "mask", "red_slot", "pseudo", "pos",
                 "uses", "mask_use", "reg", "cos_node", "store2")

    def __init__(self, op, ctype, rcls, is_bool, args, imm=0):
        self.op = op
        self.ctype = ctype
        self.rcls = rcls
        self.is_bool = is_bool
        self.args = args  # list of TV
        self.imm = imm
        self.store = None
        self.mask = None
        self.red_slot = None
        self.pseudo = False  # value lives only in a register (cos half of SINCOS)
        self.pos = -1
        self.uses = []
        self.mask_use = False
        self.reg = None
        self.cos_node = None
        self.store2 = None  # SINCOS: view the parked half is stored to


# result class of each PHILOX output form (imm)
PHILOX_CLASS = {cabi.PHILOX_UNIFORM64: T_F64, cabi.PHILOX_UNIFORM32: T_F32, cabi.PHILOX_NORMAL64: T_F64, cabi.PHILOX_INTEGER: T_I64}

_FLOAT_UNARY = {"sqrt", "sin", "cos", "tan", "sinh", "cosh", "tanh", "asin", "acos", "atan", "exp", "log", "cbrt"}
_PRED_UNARY = {"isfinite", "isinf", "isnan", "isneginf", "isposinf", "lnot"}
_CMP = {"gt", "lt", "ge", "le", "eq", "ne"}
_LOGIC = {"land", "lor", "lxor"}
_BITS = {"band", "bor", "bxor", "shl", "shr"}
_ARITH = {"add", "sub", "mul", "floordiv", "mod", "min", "max"}


def unify_cls(a, b, a_bool=False, b_bool=False):
    """Numba's scalar type unification restricted to the three classes."""
    if a == T_F64 or b == T_F64:
        return T_F64
    if a == T_F32 and b == T_F32:
        return T_F32
    if a == T_F32 or b == T_F32:
        # float32 with bool stays float32; with int64 it is float64
        other_bool = b_bool if a == T_F32 else a_bool
        return T_F32 if other_bool else T_F64
    return T_I64


class ProgramError(RuntimeError):
    pass


class ProgramLimit(ProgramError):
    """The op list would exceed a table size of the C-ABI (views, scalars, instructions, spill registers, reduction
    slots): the fuser cuts the chain in two and retries (deferred_op._run_statements)."""


class Program:
    """Lowered op list, independent of pointers and ranges."""

    def __init__(self):
        self.insns = []  # list of dict fields
        self.scalars = []  # raw uint64
        self.n_regs = 0
        self.reds = []  # list of (redop, ctype)
        self.view_written = {}
        self.uses_iota = set()


class Lowering:
    """Builds nodes from statements, then emits instructions."""

    def __init__(self, view_dtypes):
        self.view_dtypes = list(view_dtypes)  # rb dtype code per view index
        self.nodes = []
        self.scalars = []
        self._scal_index = {}
        self.view_value = {}  # view idx -> TV of the value last stored (forwarding)
        self.view_loaded = {}  # view idx -> TV of an explicit load (CSE of repeated reads)
        self.view_read_count = {}
        self.temps = {}  # temp key -> TV
        self.reds = []
        self.uses_iota = set()

    # ---- operand constructors
    def scalar(self, value):
        """Python / NumPy scalar -> typed scalar operand (ramba/ramba.py:8094-8104: scalars are
        pickled as they are; Numba then types Python float as float64, int as int64)."""
        if isinstance(value, (bool, np.bool_)):
            return self._intern(T_I64, int(bool(value)), True)
        if isinstance(value, np.floating):
            if value.dtype == np.float32:
                return self._intern(T_F32, float(value), False)
            return self._intern(T_F64, float(value), False)
        if isinstance(value, (int, np.integer)):
            v = int(value)
            if not (-(1 << 63) <= v < (1 << 63)):
                raise ProgramError("integer scalar out of int64 range")
            return self._intern(T_I64, v, False)
        if isinstance(value, float):
            return self._intern(T_F64, value, False)
        raise ProgramError("unsupported scalar operand %r" % (type(value),))

    def _intern(self, cls, value, is_bool):
        if cls == T_F64:
            bits = struct.unpack("<Q", struct.pack("<d", float(value)))[0]
        elif cls == T_F32:
            bits = struct.unpack("<I", struct.pack("<f", float(value)))[0]
        else:
            bits = int(value) & 0xFFFFFFFFFFFFFFFF
        key = (cls, bits)
        if key not in self._scal_index:
            if len(self.scalars) >= cabi.MAX_SCALARS:
                raise ProgramLimit("too many scalars in one fused op")
            self._scal_index[key] = len(self.scalars)
            self.scalars.append((cls, bits, value))
        return TV(cls, is_bool, "scal", self._scal_index[key])

    def iota(self, dim):
        self.uses_iota.add(dim)
        return TV(T_I64, False, "iota", dim)

    # ---- node construction
    def _node(self, op, ctype, rcls, is_bool, args, imm=0):
        n = Node(op, ctype, rcls, is_bool, args, imm)
        self.nodes.append(n)
        return TV(rcls, is_bool, "node", n)

    def coerce(self, tv, cls):
        """Value of `tv` in compute class `cls`."""
        if tv.cls == cls:
            return tv
        if tv.kind == "scal":
            c, bits, value = self.scalars[tv.ref]
            return self._intern(cls, int(value) if cls == T_I64 else float(value), False)
        if tv.kind in ("view", "iota"):
            # the fetch converts (C cast semantics)
            return TV(cls, False, tv.kind, tv.ref)
        return self._node("cvt", cls, cls, False, [tv], imm=tv.cls)

    def _binary(self, op, x, y):
        if op == "div":
            cls = unify_cls(x.cls, y.cls, x.is_bool, y.is_bool)
            if cls == T_I64:
                cls = T_F64
            return self._node("div", cls, cls, False, [self.coerce(x, cls), self.coerce(y, cls)])
        if op == "pow":
            if x.cls != T_I64 and y.cls == T_I64:
                return self._node("powi", x.cls, x.cls, False, [x, y])
            if x.cls == T_I64 and y.cls == T_I64:
                return self._node("powi", T_I64, T_I64, False, [x, y])
            cls = unify_cls(x.cls, y.cls)
            if cls == T_I64:
                cls = T_F64
            return self._node("pow", cls, cls, False, [self.coerce(x, cls), self.coerce(y, cls)])
        if op in ("add", "mul") and x.kind == "scal" and y.kind != "scal":
            x, y = y, x  # commutative: keep the scalar as the second operand (the specialised handlers expect it there)
        if op in _ARITH:
            cls = unify_cls(x.cls, y.cls, x.is_bool, y.is_bool)
            is_bool = False
            if op in ("min", "max") and x.is_bool and y.is_bool:
                is_bool = True
            return self._node(op, cls, cls, is_bool, [self.coerce(x, cls), self.coerce(y, cls)])
        if op in _CMP or op in _LOGIC:
            cls = unify_cls(x.cls, y.cls, x.is_bool, y.is_bool)
            return self._node(op, cls, T_I64, True, [self.coerce(x, cls), self.coerce(y, cls)])
        if op in _BITS:
            if x.cls != T_I64 or y.cls != T_I64:
                raise ProgramError("bitwise op on non-integer operands")
            return self._node(op, T_I64, T_I64, x.is_bool and y.is_bool and op in ("band", "bor", "bxor"), [x, y])
        raise ProgramError("unknown binary op " + op)

    def _unary(self, op, x):
        if op in _FLOAT_UNARY:
            cls = T_F32 if x.cls == T_F32 else T_F64
            return self._node(op, cls, cls, False, [self.coerce(x, cls)])
        if op in _PRED_UNARY:
            return self._node(op, x.cls, T_I64, True, [x])
        if op in ("abs", "neg", "square"):
            return self._node(op, x.cls, x.cls, False, [x])
        if op == "invert":
            if x.cls != T_I64:
                raise ProgramError("invert on non-integer operand")
            return self._node("invert", T_I64, T_I64, x.is_bool, [x], imm=1 if x.is_bool else 0)
        if op == "mov":
            return self._node("mov", x.cls, x.cls, x.is_bool, [x])
        raise ProgramError("unknown unary op " + op)

    def astype(self, x, code):
        """Value of x after a round trip through storage dtype `code` (what a store followed by a
        load of a live array gives), in the class of that dtype."""
        cls = dtype_class(code)
        is_bool = code == cabi.BOOL
        if x.cls == cls and code in (cabi.F64, cabi.F32, cabi.I64):
            return x
        if x.cls == cls and is_bool and x.is_bool:
            return x
        if code in (cabi.F64, cabi.F32):
            # a float storage dtype IS its compute class: the round trip is the plain class conversion
            return self.coerce(x, cls)
        tv = self._node("cvt", cls, cls, is_bool, [x], imm=x.cls | ((code + 1) << 8))
        return tv

    def build(self, expr, resolve):
        """Expression tree -> TV. `resolve(obj)` maps a fuser operand to a TV (views, temps)."""
        if isinstance(expr, E):
            op = expr.op
            if op == "where":
                c = self.build(expr.args[0], resolve)
                a = self.build(expr.args[1], resolve)
                b = self.build(expr.args[2], resolve)
                cls = unify_cls(a.cls, b.cls, a.is_bool, b.is_bool)
                if not c.is_bool and c.cls != cls:
                    # the condition is tested in ITS OWN class (`if c:` on a float 0.5 is true); only the resulting
                    # 0/1 may be converted to the class of the branches
                    c = self._node("ne", c.cls, T_I64, True, [c, self._intern(c.cls, 0, False)])
                return self._node("where", cls, cls, a.is_bool and b.is_bool,
                                  [self.coerce(c, cls), self.coerce(a, cls), self.coerce(b, cls)])
            if op == "astype":
                x = self.build(expr.args[0], resolve)
                return self.astype(x, expr.imm)
            if op == "tofloat":  # class of a "float" result dtype for an int operand (sin(int) etc.)
                x = self.build(expr.args[0], resolve)
                return self.coerce(x, T_F32 if x.cls == T_F32 else T_F64)
            if op == "philox":
                # E("philox", index, key[, bound], imm=form): one element of a random draw (include/ramba_b200.h)
                cls = PHILOX_CLASS[expr.imm]
                args = [self.coerce(self.build(expr.args[0], resolve), T_I64)]
                for a in expr.args[1:]:
                    tv = self.build(a, resolve)
                    if tv.kind != "scal" or tv.cls != T_I64:
                        raise ProgramError("philox: key and bound must be integer scalars")
                    args.append(tv)
                return self._node("philox", cls, cls, False, args, imm=expr.imm)
            if len(expr.args) == 2:
                return self._binary(op, self.build(expr.args[0], resolve), self.build(expr.args[1], resolve))
            if len(expr.args) == 1:
                return self._unary(op, self.build(expr.args[0], resolve))
            raise ProgramError("bad expression arity for " + op)
        if isinstance(expr, Iota):
            return self.iota(expr.dim)
        if isinstance(expr, TV):
            return expr
        return resolve(expr)

    # ---- statements
    def note_view_reads(self, counts):
        """Views read more than once (and not written first) are loaded once into the machine."""
        self.view_read_count = dict(counts)

    def read_view(self, vidx):
        tv = self.view(vidx)
        if tv.kind == "view" and self.view_read_count.get(vidx, 0) > 1:
            tv = self._node("mov", tv.cls, tv.cls, tv.is_bool, [tv])
            self.view_loaded[vidx] = tv
        return tv

    def _materialise(self, tv):
        """Make sure `tv` is the result of a node (so that it can carry a store)."""
        if tv.kind != "node" or tv.ref.store is not None or tv.ref.pseudo:
            tv = self._node("mov", tv.cls, tv.cls, tv.is_bool, [tv])
        return tv

    def _same_array(self, a, b):
        gids = getattr(self, "view_gids", None)
        return a == b or gids is None or gids[a] == gids[b]

    def _touched(self, nodes, vidx):
        """Does any of `nodes` read or write the array behind view `vidx`?"""
        for m in nodes:
            for a in m.args:
                if a.kind == "view" and self._same_array(a.ref, vidx):
                    return True
            if (m.store is not None and self._same_array(m.store, vidx)) or (m.store2 is not None and self._same_array(m.store2, vidx)):
                return True
        return False

    def store(self, vidx, tv, mask=None):
        code = self.view_dtypes[vidx]
        tv = self._materialise(tv)
        node = tv.ref
        if node is not self.nodes[-1]:
            # Instructions run in node order and a store runs where its node sits.  A value built by an EARLIER statement
            # (`t = a*2; b -= a; b[:] = t` with t never stored) must not carry this store back in front of statements that
            # read or write the array in between: the value is moved at THIS statement's position instead.
            i = len(self.nodes) - 1
            while self.nodes[i] is not node:
                i -= 1
            if self._touched(self.nodes[i + 1:], vidx):
                tv = self._node("mov", tv.cls, tv.cls, tv.is_bool, [tv])
                node = tv.ref
        if mask is not None:
            m = self._materialise(mask) if mask.kind != "node" else mask
            if self.nodes.index(m.ref) > self.nodes.index(node):
                # the mask has to be in a register when the storing node runs: a mask that is a stored array is loaded HERE,
                # after the value's node - the value is moved behind it (`x[m] = 0.5` with m materialised by an earlier flush)
                tv = self._node("mov", tv.cls, tv.cls, tv.is_bool, [tv])
                node = tv.ref
        node.store = vidx
        if mask is not None:
            node.mask = m.ref
            m.ref.mask_use = True
            # masked store: elements where the mask is false keep their old value -> no forwarding
            self.view_value.pop(vidx, None)
            self.view_loaded.pop(vidx, None)
            return
        # value later reads of this view see: the stored value after rounding to the dtype
        self.view_loaded.pop(vidx, None)
        cls = dtype_class(code)
        exact = (tv.cls == cls and code in (cabi.F64, cabi.F32, cabi.I64)) or (code == cabi.BOOL and tv.is_bool)
        if exact:
            self.view_value[vidx] = tv
        else:
            self.view_value[vidx] = ("lazy", tv, code)

    def view(self, vidx):
        """Current value of a view element: forwarded if this fused op already stored to it."""
        v = self.view_value.get(vidx)
        if v is not None:
            if isinstance(v, tuple):
                _, tv, code = v
                v = self.astype(tv, code)
                self.view_value[vidx] = v
            return v
        if vidx in self.view_loaded:
            return self.view_loaded[vidx]
        code = self.view_dtypes[vidx]
        return TV(dtype_class(code), code == cabi.BOOL, "view", vidx)

    def reduce(self, redop, tv):
        """Global / axis reduction stage 1: acc = acc (op) value (ramba/ramba.py:5798-5814).
        Floats accumulate in float64 (the reference's scalar accumulator is seeded with a Python
        int and unifies to float64, SURVEY §8a a10), integers and bools in int64."""
        cls = T_I64 if tv.cls == T_I64 else T_F64
        if len(self.reds) >= cabi.MAX_REDS:
            raise ProgramLimit("too many reductions in one fused op")
        slot = len(self.reds)
        self.reds.append((redop, cls))
        x = self.coerce(tv, cls)
        n = Node("red", cls, cls, False, [x], imm=redop)
        n.red_slot = slot
        self.nodes.append(n)
        return slot

    # ---- peepholes
    def _fuse_sincos(self):
        """sin(x) and cos(x) of the same operand share one range reduction: the first of the pair
        becomes SINCOS (imm 0: acc = sin, imm 1: acc = cos) and parks the other half in a spill
        register that the second reads back."""

        def key(n):
            a = n.args[0]
            return (n.ctype, a.kind, id(a.ref) if a.kind == "node" else a.ref)

        first = {}
        i = 0
        while i < len(self.nodes):
            n = self.nodes[i]
            i += 1
            if n.op not in ("sin", "cos") or n.ctype not in (T_F64, T_F32):
                continue
            k = key(n)
            f = first.get(k)
            if f is None or f.op == n.op or f.cos_node is not None:
                first.setdefault(k, n)
                continue
            # f computes both halves
            f.imm = 0 if f.op == "sin" else 1
            f.op = "sincos"
            p = Node("cospart", f.ctype, f.rcls, False, [TV(f.rcls, False, "node", f)])
            p.pseudo = True
            f.cos_node = p
            self.nodes.insert(self.nodes.index(f) + 1, p)
            i += 1
            # the second node becomes a read-back of the parked half ...
            n.op = "mov"
            n.args = [TV(f.rcls, False, "node", p)]
            # ... unless all it does is store the value in its own dtype: then SINCOS stores the parked
            # half itself and every later use reads the parked register directly
            own = {T_F64: cabi.F64, T_F32: cabi.F32}[f.rcls]
            between = self.nodes[self.nodes.index(p) + 1:self.nodes.index(n)]
            if n.mask is None and not n.mask_use and (n.store is None or (self.view_dtypes[n.store] == own
                                                                          and not self._touched(between, n.store))):
                # (moving the store of the second half up to the SINCOS is only right if nothing in between reads or writes
                # that array)
                f.store2 = n.store
                n.store = None
                for m in self.nodes:
                    for a in m.args:
                        if a.kind == "node" and a.ref is n:
                            a.ref = p
                    if m.mask is n:
                        m.mask = p

    def _drop_dead_stores(self):
        """A store is dead when a later unmasked store of the same fused op overwrites the same view and no
        read in between can observe it (`a += 1` ten times in one flush writes `a` once; the reference's
        fused loop also stores every time, but its stores hit the cache line it just wrote).
        view_gids (set by the fuser) tells which views alias the same array; without it any view read is
        assumed to observe every pending store."""
        gids = getattr(self, "view_gids", None)
        pending = {}  # view idx -> node whose store is not yet known to be observed
        for n in self.nodes:
            for a in n.args:
                if a.kind == "view":
                    for v in list(pending):
                        if gids is None or v == a.ref or gids[v] == gids[a.ref]:
                            pending.pop(v)
            if n.store2 is not None:
                pending.pop(n.store2, None)
            if n.store is not None:
                prev = pending.get(n.store)
                if prev is not None and n.mask is None:
                    prev.store = None
                    prev.mask = None
                pending[n.store] = n

    _LEAN_OPS = {"mov", "add", "sub", "mul", "div", "neg", "abs", "square", "min", "max", "cvt", "red"}

    @staticmethod
    def _fuse_muladd(nodes):
        """`x + s*y`, `x - s*y`, `s*y - x`: when the product has no other use it is folded into the sum as a
        three-operand instruction (MULADD / MULSUB / MULRSUB; product and sum still round separately), so that the
        running sum stays in the accumulator instead of being parked in a spill register around the multiplication
        - the shape of every weighted stencil term (ramba/ramba.py:8146-8188).  Applied only to op lists made of
        plain float arithmetic (the ones the tile / stream kernels of the library take); anything with
        transcendentals, integers, masks or index operands keeps the two-operand form its specialised handlers
        expect."""
        for n in nodes:
            if n.pseudo or n.op not in Lowering._LEAN_OPS or n.ctype == T_I64 or n.mask is not None or n.mask_use:
                return nodes
            if n.op == "cvt" and ((n.imm >> 8) != 0 or (n.imm & 0xFF) == T_I64):
                return nodes
            if any(a.kind == "iota" for a in n.args):
                return nodes
        uses = {}
        for n in nodes:
            for a in n.args:
                if a.kind == "node":
                    uses[id(a.ref)] = uses.get(id(a.ref), 0) + 1

        def product(tv, n):
            if tv.kind != "node":
                return None
            m = tv.ref
            if (m.op != "mul" or m.ctype != n.ctype or uses.get(id(m), 0) != 1 or m.store is not None
                    or m.red_slot is not None or m.store2 is not None):
                return None
            return m

        dropped = set()
        for n in nodes:
            if n.op not in ("add", "sub") or len(n.args) != 2:
                continue
            x, y = n.args
            m = product(y, n)
            if m is not None:
                n.op = "muladd" if n.op == "add" else "mulsub"
                n.args = [x, m.args[0], m.args[1]]
                dropped.add(id(m))
                continue
            m = product(x, n)
            if m is not None:
                n.op = "muladd" if n.op == "add" else "mulrsub"
                n.args = [y, m.args[0], m.args[1]]
                dropped.add(id(m))
        return [n for n in nodes if id(n) not in dropped]

    # ---- emission
    def finish(self):
        self._fuse_sincos()
        self._drop_dead_stores()
        nodes = self.nodes
        # dead code elimination (values nobody uses and that have no side effect)
        live = set()

        def mark(n):
            if id(n) in live:
                return
            live.add(id(n))
            for a in n.args:
                if a.kind == "node":
                    mark(a.ref)
            if n.mask is not None:
                mark(n.mask)

        for n in nodes:
            if n.store is not None or n.red_slot is not None or n.store2 is not None:
                mark(n)
                if n.store2 is not None and n.cos_node is not None:
                    mark(n.cos_node)
        nodes = [n for n in nodes if id(n) in live]
        # a SINCOS whose parked half died is a plain sin / cos again
        for n in nodes:
            if n.op == "sincos" and (n.cos_node is None or id(n.cos_node) not in live):
                n.op = "sin" if n.imm == 0 else "cos"
                n.imm = 0
                n.cos_node = None

        nodes = self._fuse_muladd(nodes)
        # emission positions (pseudo nodes emit nothing)
        pos = 0
        for n in nodes:
            if n.pseudo:
                n.pos = -1
            else:
                n.pos = pos
                pos += 1
        if pos > cabi.MAX_INSNS:
            raise ProgramLimit("fused op too long (%d instructions)" % pos)
        # uses
        for n in nodes:
            n.uses = []
        for n in nodes:
            if n.pseudo:
                continue
            for a in n.args:
                if a.kind == "node":
                    a.ref.uses.append(n.pos)
            if n.mask is not None:
                n.mask.uses.append(n.pos)
        # pseudo nodes forward their uses' positions for liveness; their value is in a register

        # register allocation
        free = list(range(cabi.MAX_REGS))
        n_regs = 0
        release = {}  # pos -> [regs]
        prog = Program()
        prog.reds = list(self.reds)
        prog.uses_iota = set(self.uses_iota)

        def alloc(last_use):
            nonlocal n_regs
            if not free:
                raise ProgramLimit("fused op needs more than %d spill registers" % cabi.MAX_REGS)
            r = free.pop(0)
            n_regs = max(n_regs, r + 1)
            release.setdefault(last_use, []).append(r)
            return r

        emitted = -1
        for n in nodes:
            if n.pseudo:
                continue
            # operands
            fields = dict(op=OP[n.op.upper()], ctype=n.ctype, a_kind=K_NONE, a_idx=0, b_kind=K_NONE, b_idx=0,
                          c_kind=K_NONE, c_idx=0, st_reg=NOSTORE, st_view=NOSTORE, st2=NOSTORE, mask_reg=NOSTORE,
                          imm=n.imm)
            names = ("a", "b", "c")
            for i, a in enumerate(n.args):
                if a.kind == "node":
                    src = a.ref
                    if src.pseudo:
                        kind, idx = K_REG, src.reg
                    elif src.pos == n.pos - 1 and src.pos == emitted:
                        kind, idx = K_ACC, 0
                        if src.reg is not None:
                            kind, idx = K_ACC, 0
                    else:
                        if src.reg is None:
                            raise ProgramError("internal: value not in a register")
                        kind, idx = K_REG, src.reg
                elif a.kind == "view":
                    kind, idx = K_VIEW, a.ref
                elif a.kind == "scal":
                    kind, idx = K_SCAL, a.ref
                else:
                    kind, idx = K_IOTA, a.ref
                fields[names[i] + "_kind"] = kind
                fields[names[i] + "_idx"] = idx
            if n.op == "red":
                fields["b_idx"] = n.red_slot
            if n.op == "sincos" and n.store2 is not None:
                fields["c_kind"] = K_VIEW
                fields["c_idx"] = n.store2
                prog.view_written[n.store2] = True
            if n.mask is not None:
                if n.mask.reg is None:
                    raise ProgramError("internal: mask not in a register")
                fields["mask_reg"] = n.mask.reg
            # does the result need a register?
            needs_reg = n.mask_use or any(u != n.pos + 1 for u in n.uses)
            if needs_reg and n.uses:
                n.reg = alloc(max(n.uses))
                fields["st_reg"] = n.reg
            elif n.mask_use and n.uses:
                n.reg = alloc(max(n.uses))
                fields["st_reg"] = n.reg
            if n.op == "sincos":
                c = n.cos_node
                cu = []
                for m in nodes:
                    if m.pseudo:
                        continue
                    for a in m.args:
                        if a.kind == "node" and a.ref is c:
                            cu.append(m.pos)
                    if m.mask is c:
                        cu.append(m.pos)
                c.reg = alloc(max(cu) if cu else n.pos)
                fields["st2"] = c.reg
            if n.store is not None:
                fields["st_view"] = n.store
                prog.view_written[n.store] = True
            prog.insns.append(fields)
            emitted = n.pos
            for r in release.pop(n.pos, []):
                free.append(r)
                free.sort()
        prog.scalars = [bits for (_, bits, _) in self.scalars]
        prog.n_regs = n_regs
        return prog
