"""Elementwise ops at their edge values, against references that do not come from the oracle.

Every expected value here is computed independently of oracle/vm.py: with Python integers and `math` for the integer and
conversion rules, NumPy where NumPy defines the result, a Python loop for min / max (builtins.min / max), and mpmath at
200 bits for the library functions.  The CPU tests run every case on the NumPy oracle; the -m gpu tests run the same
cases on the H100, on the 1-D kernels and on the N-d kernel (a strided 2-D view), and check that each case reached the
path it is named for.

Exact families compare bit for bit (NaN as NaN, any payload; zeros and infinities with their sign):
  A  the int64 class: `//`, `%` (zero divisors give 0), `**` (Numba's int_power), wrapping `+ - *`, multiply-add, abs and
     negation of INT64_MIN, shifts (NumPy's rule outside [0, 63]), `~`, `not`, comparisons, narrowing stores, and the
     int32 / int16 / int8 / unsigned sources;
  B  the float64 and float32 classes: `//`, `%`, `/` and `**` specials, sqrt, subnormals kept through + - * / on every
     operand kind of the specialised handlers, comparisons, logical ops, where with a NaN condition, the is* tests and
     min / max with NaN and signed zeros;
  C  conversions: float -> integer on every device path (astype to int64, astype to a narrower integer feeding a later
     instruction, a float result stored to an integer view) under one rule - NaN, +-inf and |x| >= 2^63 give INT64_MIN,
     other values truncate, narrower integers keep the low bits - and int64 -> float64 / float32 and float64 -> float32
     rounding (ties to even, overflow, subnormal results).
Family D holds tan, sinh, cosh, tanh, asin, acos, atan, exp, log, cbrt, sqrt and pow to CUDA's documented maximum ulp
errors (ULP_BOUND) in the float64 and float32 classes, and float32 arrays computed in float64 to half an ulp of float32
plus 2^-28 relative; their specials compare bit for bit.

Each value of families A-C sits at every element position of a thread (k = 0..V-1 of the V = 8 1-D tile and the V = 4
N-d tile) and in a ragged last tile: value i of an odd-length list fills the elements e with e % len == i."""
import functools
import itertools
import json
import math
import os
import subprocess
import sys

import mpmath
import numpy as onp
import pytest
from mpmath import libmp

from test_sincos_accuracy import ulp_error, rounded_bound

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")

PREC = 200
TILE = 256 * 8    # the 1-D kernels' tile; the N-d kernel's (256 * 4) divides it
RAGGED = 999      # elements in the last, partial tile
ND_WIDTH = 1000   # row length of the N-d placement (a strided 2-D view that does not collapse to 1-D)
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1

# CUDA C++ Programming Guide, CUDA 12.x, appendix "Mathematical Functions", tables "Single-Precision" and
# "Double-Precision Mathematical Standard Library Functions with Maximum ULP Error": the maximum ulp error of each
# function over its full range (0 = correctly rounded, checked here as at most half an ulp).  Double-precision rows:
# exp, log, cbrt, cosh, tanh 1; sinh, tan, asin, acos, atan, pow 2; sqrt 0 (IEEE round-to-nearest).  Single-precision
# rows: logf, cbrtf 1; expf, coshf, tanhf, asinf, acosf, atanf 2; sinhf 3; tanf, powf 4; sqrtf 0 (the default
# -prec-sqrt=true).
ULP_BOUND = {
    "float64": {"exp": 1, "log": 1, "cbrt": 1, "cosh": 1, "tanh": 1, "sinh": 2, "tan": 2, "asin": 2, "acos": 2, "atan": 2,
                "pow": 2, "sqrt": 0},
    "float32": {"log": 1, "cbrt": 1, "exp": 2, "cosh": 2, "tanh": 2, "asin": 2, "acos": 2, "atan": 2, "sinh": 3, "tan": 4,
                "pow": 4, "sqrt": 0},
}
# Findings: results above the documented bound, measured on an H100 80GB HBM3 (CUDA 12.9).  Each is held to the
# largest error measured over this file's arguments, so that any growth fails, and listed in DESIGN section 6.
FINDINGS = {("cosh", "float64"): 1.04, ("tanh", "float64"): 1.06}  # measured 1.035 and 1.052 ulp against a bound of 1


# ---- independent rules ------------------------------------------------------------------------------------------------
def wrap(v, dtype=onp.int64):
    """Python int v kept to the low bits of an integer dtype (two's complement), or v != 0 for bool"""
    dt = onp.dtype(dtype)
    if dt == onp.bool_:
        return int(v != 0)
    bits = 8 * dt.itemsize
    v &= (1 << bits) - 1
    if dt.kind == "i" and v >> (bits - 1):
        v -= 1 << bits
    return v


def f2i(x):
    """float -> int64 on every path: NaN, +-inf and |x| >= 2^63 give INT64_MIN, anything else truncates toward zero"""
    x = float(x)
    return math.trunc(x) if abs(x) < 2.0 ** 63 else I64_MIN


def py_floordiv(a, b):
    return 0 if b == 0 else wrap(a // b)


def py_mod(a, b):
    return 0 if b == 0 else a % b


def int_power(a, e):
    """Numba's int_power for int64: square-and-multiply with wrapping (the exact power, wrapped); a negative exponent
    gives 1 for a base of 1, +-1 for -1 and 0 for any other base (0 included) - a pinned choice, Numba itself divides"""
    if e < 0:
        return 1 if a == 1 else (-1 if e & 1 else 1) if a == -1 else 0
    return wrap(pow(a, e, 1 << 64))


def shl(a, c):
    return wrap(a << c) if 0 <= c < 64 else 0


def shr(a, c):
    return a >> c if 0 <= c < 64 else (-1 if a < 0 else 0)


def py_min(a, b):  # builtins.min(a, b): b only when b < a, so a NaN survives only in a
    return b if b < a else a


def py_max(a, b):
    return b if b > a else a


def to_f32_once(v):
    """Python int v rounded once to float32 (ties to even)"""
    return onp.float32(libmp.to_float(libmp.from_int(int(v), 24, libmp.round_nearest)))


# ---- value sets -------------------------------------------------------------------------------------------------------
INTS = [0, 1, -1, 2, -2, 3, -3, 7, -7, 1 << 31, -(1 << 31) - 1, 12345678901, -98765, 1 << 62, -(1 << 62), I64_MAX, I64_MIN]
POW_BASES = [0, 1, -1, 2, -2, 3, -3, 7, 1 << 31, I64_MIN, I64_MAX]
POW_EXPS = [0, 1, 2, 62, 63, 64, -1, -2, -3]
SHIFT_COUNTS = [0, 1, 62, 63, 64, 65, -1, -64, 200]
BOUNDARIES = sorted({s * ((1 << k) + d) for k in (7, 8, 15, 16, 31, 32, 62) for d in (-1, 0, 1) for s in (1, -1)} | {0, I64_MAX, I64_MIN})


def floats(dtype):
    f = onp.finfo(dtype)
    sub = float(f.smallest_subnormal)
    vals = [0.0, -0.0, sub, -sub, float(f.tiny), -float(f.tiny), float(f.tiny) * 0.75, 1.0, -1.0, 1.5, -2.5, float(f.max),
            -float(f.max) / 3, onp.inf, -onp.inf, onp.nan, 7.0]
    return onp.array(vals, dtype=dtype)


CASTS = [onp.nan, onp.inf, -onp.inf, 2.0 ** 63, -2.0 ** 63, 2.0 ** 63 - 1024, -(2.0 ** 63 - 1024), 2.0 ** 31, -2.0 ** 31,
         2.0 ** 31 + 0.5, 2.0 ** 31 - 0.5, -0.5, -0.0, 0.0, 1e19, -1e19, 5e-324, -5e-324, 3e9, -3e9, 1.5, -1.5, 255.9, -128.5,
         65535.5, 32768.25, 4294967295.75, 2.0 ** 53 + 2, 1e-300]
INT_TO_FLOAT = [(1 << 53) + 1, (1 << 53) + 3, -((1 << 53) + 1), (1 << 24) + 1, (1 << 24) + 3, (1 << 60) + (1 << 36) + 1,
                (1 << 60) + (1 << 36), I64_MAX, I64_MIN, 0, -1, 1 << 62, (1 << 63) - (1 << 39)]
TO_F32 = [3.5e38, -3.5e38, 3.4028235677973366e38, 3.4028234663852886e38, 1e-40, -1e-40, 1e-45, 7e-46, 7.1e-46, 1e-50, -0.0,
          1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24, 1 - 2.0 ** -25, onp.nan, onp.inf, -onp.inf, 16777217.0, 0.1]


def spread(columns):
    """Columns of equal odd length m -> arrays of m * TILE + RAGGED elements where element e holds row e % m: every row
    at every element position of a thread, and some in the ragged last tile.  Returns (arrays, row of each element)."""
    m = len(columns[0])
    if m % 2 == 0:
        columns = [list(c) + [c[0]] for c in columns]
        m += 1
    row = onp.arange(m * TILE + RAGGED) % m
    return [onp.asarray(c)[row] for c in columns], row


def pairs(xs, ys):
    p = list(itertools.product(xs, ys))
    return [a for a, _ in p], [b for _, b in p]


# ---- cases ------------------------------------------------------------------------------------------------------------
class Case:
    """inputs: name -> (values, dtype); run(rb, X) -> [rb arrays]; want(x) -> [expected NumPy arrays] from the flat
    inputs; ops: opcodes that must appear in the op lists it runs; check(insns, views): the path it is named for"""

    def __init__(self, family, name, inputs, run, want, ops=(), check=None):
        self.family, self.name, self.inputs, self.run, self.want, self.ops, self.check = family, name, inputs, run, want, ops, check


def _elementwise(fn, *xs, out=onp.int64):
    return onp.array([fn(*v) for v in zip(*[x.tolist() for x in xs])], dtype=out)


def recip_div(a, b):
    """`a / b` of arrays is `a * (1.0 / b)`, the reciprocal a float64 temporary (the reference's array_binop turns every
    true division into a multiplication by the reciprocal): 0 / 5e-324 is NaN and 5e-324 / 5e-324 is inf"""
    return (a.astype(onp.float64) * (1.0 / b.astype(onp.float64))).astype(a.dtype)


def _np_bits(f, dt):
    def want(x):
        with onp.errstate(all="ignore"):
            return [onp.asarray(f(x), dtype=dt)]
    return want


def _through_cvt(plan, insns, views):
    return any(op == "CVT" and imm >> 8 for op, cls, imm, sv in insns)


def _float_store_to_int(plan, insns, views):
    return any(cls in ("F64", "F32") and sv is not None and views[sv] not in ("F64", "F32") for op, cls, imm, sv in insns)


def _generic_pcs(plan):
    for f in plan.split():
        if f.startswith("generic="):
            return {int(i) for i in f[len("generic="):].split(",")}
    return set()


def _plain_cvt_to_int(plan, insns, views):
    """a CVT float class -> int64 without a storage round trip (imm >> 8 == 0); on the 1-D kernel through its
    specialised handler (h_cvt), not the generic decode"""
    pcs = [pc for pc, (op, cls, imm, sv) in enumerate(insns) if op == "CVT" and cls == "I64" and imm >> 8 == 0 and (imm & 0xFF) in (0, 1)]
    if " ndim=1 " in plan:
        pcs = [pc for pc in pcs if pc not in _generic_pcs(plan)]
    return bool(pcs)


def cases():
    import ramba_b200 as rb

    out = []
    # ---- A: the int64 class
    a, b = pairs(INTS, INTS)
    ab = {"a": (a, onp.int64), "b": (b, onp.int64)}
    for name, f, rf, op in (("//", lambda X: X["a"] // X["b"], py_floordiv, "FLOORDIV"), ("%", lambda X: X["a"] % X["b"], py_mod, "MOD"),
                            ("+", lambda X: X["a"] + X["b"], lambda p, q: wrap(p + q), "ADD"),
                            ("-", lambda X: X["a"] - X["b"], lambda p, q: wrap(p - q), "SUB"),
                            ("*", lambda X: X["a"] * X["b"], lambda p, q: wrap(p * q), "MUL"),
                            ("<", lambda X: X["a"] < X["b"], lambda p, q: p < q, "LT"),
                            (">=", lambda X: X["a"] >= X["b"], lambda p, q: p >= q, "GE"),
                            ("==", lambda X: X["a"] == X["b"], lambda p, q: p == q, "EQ"),
                            ("logical_xor", lambda X: rb.logical_xor(X["a"], X["b"]), lambda p, q: (p != 0) != (q != 0), "LXOR")):
        rt = onp.bool_ if op in ("LT", "GE", "EQ", "LXOR") else onp.int64
        out.append(Case("A", "int64 " + name, ab, lambda rb, X, f=f: [f(X)], lambda x, rf=rf, rt=rt: [_elementwise(rf, x["a"], x["b"], out=rt)], (op,)))
    out.append(Case("A", "int64 a + b * b", ab, lambda rb, X: [X["a"] + X["b"] * X["b"]],
                    lambda x: [_elementwise(lambda p, q: wrap(p + wrap(q * q)), x["a"], x["b"])], ("MUL", "ADD")))
    one = {"a": (INTS, onp.int64)}
    for name, f, rf, op in (("abs", lambda X: abs(X["a"]), lambda p: wrap(abs(p)), "ABS"), ("neg", lambda X: -X["a"], lambda p: wrap(-p), "NEG"),
                            ("~", lambda X: ~X["a"], lambda p: ~p, "INVERT"), ("not", lambda X: rb.logical_not(X["a"]), lambda p: p == 0, "LNOT"),
                            ("abs(a) * 1", lambda X: abs(X["a"]) * 1, lambda p: wrap(abs(p)), "ABS")):
        rt = onp.bool_ if op == "LNOT" else onp.int64
        out.append(Case("A", "int64 " + name, one, lambda rb, X, f=f: [f(X)], lambda x, rf=rf, rt=rt: [_elementwise(rf, x["a"], out=rt)], (op,)))
    pa, pe = pairs(POW_BASES, POW_EXPS)
    out.append(Case("A", "int64 **", {"a": (pa, onp.int64), "b": (pe, onp.int64)}, lambda rb, X: [X["a"] ** X["b"]],
                    lambda x: [_elementwise(int_power, x["a"], x["b"])], ("POWI",)))
    sa, sc = pairs(INTS, SHIFT_COUNTS)
    sh = {"a": (sa, onp.int64), "b": (sc, onp.int64)}
    out.append(Case("A", "int64 <<", sh, lambda rb, X: [X["a"] << X["b"]], lambda x: [_elementwise(shl, x["a"], x["b"])], ("SHL",)))
    out.append(Case("A", "int64 >>", sh, lambda rb, X: [X["a"] >> X["b"]], lambda x: [_elementwise(shr, x["a"], x["b"])], ("SHR",)))
    for dt in (onp.int32, onp.int16, onp.int8, onp.uint8, onp.uint16, onp.uint32, onp.bool_):
        def run(rb, X, dt=dt):
            o = rb.zeros(X["a"].shape, dtype=dt)
            o[...] = X["a"]
            return [o]
        out.append(Case("A", "int64 stored to %s" % onp.dtype(dt).name, {"a": (BOUNDARIES, onp.int64)}, run,
                        lambda x, dt=dt: [_elementwise(lambda p: wrap(p, dt), x["a"], out=dt)], ("MOV",), _int_store_narrow))
    for dt in (onp.int32, onp.int16, onp.int8, onp.uint8, onp.uint16, onp.uint32):
        vals = sorted({wrap(v, dt) for v in INTS + BOUNDARIES})
        pa, pb = pairs(vals[:: max(1, len(vals) // 12)], vals[:: max(1, len(vals) // 12)])
        for name, f, rf, op in (("//", lambda X: X["a"] // X["b"], py_floordiv, "FLOORDIV"), ("%", lambda X: X["a"] % X["b"], py_mod, "MOD"),
                                ("*", lambda X: X["a"] * X["b"], lambda p, q: p * q, "MUL"), ("-", lambda X: X["a"] - X["b"], lambda p, q: p - q, "SUB")):
            def want(x, rf=rf):
                return [onp.array([rf(p, q) for p, q in zip(x["a"].tolist(), x["b"].tolist())], dtype=object)]
            out.append(Case("A", "%s %s" % (onp.dtype(dt).name, name), {"a": (pa, dt), "b": (pb, dt)}, lambda rb, X, f=f: [f(X)], want, (op,)))

    # ---- B: the float classes
    for dt in (onp.float64, onp.float32):
        n = onp.dtype(dt).name
        fa, fb = pairs(floats(dt), floats(dt))
        ab = {"a": (fa, dt), "b": (fb, dt)}
        for name, f, nf, op in (("//", lambda X: X["a"] // X["b"], onp.floor_divide, "FLOORDIV"), ("%", lambda X: X["a"] % X["b"], onp.mod, "MOD"),
                                ("/", lambda X: X["a"] / X["b"], recip_div, "MUL"), ("+", lambda X: X["a"] + X["b"], onp.add, "ADD"),
                                ("-", lambda X: X["a"] - X["b"], onp.subtract, "SUB"), ("*", lambda X: X["a"] * X["b"], onp.multiply, "MUL"),
                                ("<", lambda X: X["a"] < X["b"], onp.less, "LT"), ("!=", lambda X: X["a"] != X["b"], onp.not_equal, "NE"),
                                ("<=", lambda X: X["a"] <= X["b"], onp.less_equal, "LE"),
                                ("logical_and", lambda X: rb.logical_and(X["a"], X["b"]), onp.logical_and, "LAND"),
                                ("logical_or", lambda X: rb.logical_or(X["a"], X["b"]), onp.logical_or, "LOR")):
            out.append(Case("B", "%s %s" % (n, name), ab, lambda rb, X, f=f: [f(X)], lambda x, nf=nf: _np_bits(lambda y: nf(y["a"], y["b"]), None)(x), (op,)))
        out.append(Case("B", "%s where(a, b, 2)" % n, ab, lambda rb, X: [rb.where(X["a"], X["b"], X["b"] * 2)],
                        lambda x: _np_bits(lambda y: onp.where(y["a"] != 0, y["b"], y["b"] * y["b"].dtype.type(2)), None)(x), ("WHERE",)))
        for name, f in (("minimum", rb.minimum), ("maximum", rb.maximum)):
            rf = py_min if name == "minimum" else py_max
            out.append(Case("B", "%s %s" % (n, name), ab, lambda rb, X, f=f: [f(X["a"], X["b"])],
                            lambda x, rf=rf: [_elementwise(rf, x["a"], x["b"], out=x["a"].dtype)], ("MIN" if name == "minimum" else "MAX",)))
        one = {"a": (floats(dt), dt)}
        for name in ("isfinite", "isinf", "isnan", "isneginf", "isposinf", "sqrt", "abs", "negative", "logical_not"):
            f = {"abs": lambda X: abs(X["a"]), "negative": lambda X: -X["a"]}.get(name, lambda X, name=name: getattr(rb, name)(X["a"]))
            nf = getattr(onp, name)
            out.append(Case("B", "%s %s" % (n, name), one, lambda rb, X, f=f: [f(X)], lambda x, nf=nf: _np_bits(lambda y: nf(y["a"]), None)(x)))
        # pow at the C99 Annex F specials
        inf, nan = onp.inf, onp.nan
        big = 1100.0 if dt == onp.float64 else 200.0
        pw = [(x, y) for x in floats(dt) for y in (0.0, -0.0)] + [(1.0, nan), (1.0, inf), (-1.0, inf), (-1.0, -inf), (-0.0, -3.0), (0.0, -3.0),
             (-0.0, 3.0), (-0.0, -2.0), (-0.0, -inf), (0.0, -inf), (-8.0, 1.0 / 3), (-2.0, 0.5), (2.0, big), (2.0, -big), (0.5, big), (-2.0, big + 1),
             (-2.0, big), (inf, -1.0), (-inf, 3.0), (-inf, -3.0), (-inf, 2.0), (0.5, inf), (0.5, -inf), (2.0, inf), (2.0, -inf), (nan, 0.0),
             (nan, 1.0), (4.0, 0.5), (-inf, 0.5), (1.0, -inf)]
        out.append(Case("B", "%s ** specials" % n, {"a": ([p for p, _ in pw], dt), "b": ([q for _, q in pw], dt)},
                        lambda rb, X: [X["a"] ** X["b"]], lambda x: _np_bits(lambda y: onp.power(y["a"], y["b"]), None)(x), ("POW",)))
        # subnormal operands and results through each operand kind of the specialised + - * / handlers
        sub = float(onp.finfo(dt).smallest_subnormal)
        tiny = float(onp.finfo(dt).tiny)
        sa = [sub, 3 * sub, tiny, tiny * 0.5, -tiny * 0.25, tiny * 1.5, 2 * tiny, -sub, tiny * 0.75]
        sb = [sub, sub, tiny * 0.75, tiny * 0.25, tiny * 0.5, -tiny, -tiny * 1.25, 5 * sub, -tiny]
        sab = {"a": (sa, dt), "b": (sb, dt)}
        s = dt(2.0 ** -10)

        def sub_want(x, s=s):
            a_, b_ = x["a"], x["b"]
            return [a_ + b_, a_ - b_, a_ * s, b_ / dt(4.0), (a_ + b_) * dt(0.5), onp.sqrt(onp.abs(a_)), a_ * dt(1.0) - b_]

        out.append(Case("B", "%s subnormals" % n, sab, lambda rb, X, s=s: [X["a"] + X["b"], X["a"] - X["b"], X["a"] * s, X["b"] / dt(4.0),
                                                                         (X["a"] + X["b"]) * dt(0.5), rb.sqrt(abs(X["a"])), X["a"] * dt(1.0) - X["b"]],
                        sub_want, ("ADD", "SUB", "MUL")))
    sa64 = [float(v) for v in onp.array([1e-45, 3e-45, 1.2e-38, 6e-39, 1.4e-45, 2.5e-40, 1e-40, 1.5e-38, 5e-44], dtype=onp.float32)]
    sb64 = [1e-310, -2e-310, 5e-324, -1e-320, 2e-308, 3e-310, -1e-45, 1e-300, -5e-324]
    # a float32 view read as float64 (the staged f32-as-f64 load): no rounding, nothing flushed
    out.append(Case("B", "float32 view + float64 view", {"a": (sa64, onp.float32), "b": (sb64, onp.float64)},
                    lambda rb, X: [X["a"] + X["b"], X["a"] * 1.0, X["b"] - X["a"]],
                    lambda x: [x["a"].astype(onp.float64) + x["b"], x["a"], x["b"] - x["a"].astype(onp.float64)], ("ADD", "SUB")))

    # ---- C: conversions
    for dt in (onp.float64, onp.float32):
        n = onp.dtype(dt).name
        with onp.errstate(over="ignore"):
            src = sorted(set(onp.array(CASTS, dtype=dt).tolist()), key=lambda v: (math.isnan(v), v))
        cx = {"a": (src, dt)}
        for it in (onp.int64, onp.int32, onp.int16, onp.int8, onp.uint8, onp.uint16, onp.uint32, onp.bool_):
            itn = onp.dtype(it).name

            def conv(p, it=it):
                return int(p != 0) if it == onp.bool_ else wrap(f2i(p), it)

            # t is stored (a float MOV to an integer view) and read back by a later instruction of the same op list: a
            # CVT through t's storage dtype (a temporary that dies unobserved would stay un-rounded, as in the reference)
            def thr_want(x, conv=conv, it=it):
                v = [conv(p) for p in x["a"].tolist()]
                return [onp.array(v, dtype=it), onp.array([q + 1 for q in v], dtype=object)]

            out.append(Case("C", "%s astype %s, + 1" % (n, itn), cx, lambda rb, X, it=it: (lambda t: [t, t + 1])(X["a"].astype(it)), thr_want,
                            ("ADD",), lambda p, ii, views: _through_cvt(p, ii, views) and _float_store_to_int(p, ii, views)))

            def store(rb, X, it=it):
                o = rb.zeros(X["a"].shape, dtype=it)
                o[...] = X["a"] * X["a"].dtype.type(1.0)
                return [o]

            out.append(Case("C", "%s * 1 stored to %s" % (n, itn), cx, store, lambda x, conv=conv, it=it: [_elementwise(conv, x["a"], out=it)],
                            ("MUL",), _float_store_to_int))
        # a masked float assignment into an int64 temporary that never leaves the registers: the float value is
        # converted by a plain CVT (no storage round trip), on the 1-D kernel through its specialised handler
        k = len(src)
        mx = {"a": (src, dt), "i": ([7 * j - 50 for j in range(k)], onp.int64), "m": ([j % 4 != 3 for j in range(k)], onp.bool_)}

        def masked(rb, X, dt=dt):
            t = X["i"] * 2
            t[X["m"]] = X["a"] * dt(1.0)
            r = t + 1
            del t
            return [r]

        out.append(Case("C", "%s masked into a dead int64 temporary, + 1" % n, mx, masked,
                        lambda x: [_elementwise(lambda p, q, c: wrap((f2i(p) if c else 2 * q) + 1), x["a"], x["i"], x["m"])],
                        ("CVT", "WHERE"), _plain_cvt_to_int))
    ix = {"a": (INT_TO_FLOAT, onp.int64)}
    out.append(Case("C", "int64 astype float64", ix, lambda rb, X: [X["a"].astype(onp.float64), X["a"] * 1.0],
                    lambda x: [onp.array([float(v) for v in x["a"].tolist()])] * 2))
    out.append(Case("C", "int64 astype float32", ix, lambda rb, X: [X["a"].astype(onp.float32)],
                    lambda x: [onp.array([to_f32_once(v) for v in x["a"].tolist()], dtype=onp.float32)]))
    out.append(Case("C", "float64 astype float32", {"a": (TO_F32, onp.float64)}, lambda rb, X: [X["a"].astype(onp.float32)],
                    lambda x: _np_bits(lambda y: y["a"].astype(onp.float32), None)(x)))
    return out


# ---- running a case ---------------------------------------------------------------------------------------------------
def flat_inputs(case, placement):
    """flat NumPy inputs of the case as the placement lays them out"""
    names = list(case.inputs)
    with onp.errstate(over="ignore"):
        cols, _ = spread([onp.asarray(case.inputs[k][0], dtype=object if case.inputs[k][1] == onp.int64 else None) for k in names])
        flat = {k: onp.asarray(c.tolist() if c.dtype == object else c).astype(case.inputs[k][1]) for k, c in zip(names, cols)}
    if placement == "nd":
        rows = -(-flat[names[0]].size // ND_WIDTH)
        flat = {k: onp.resize(x, rows * ND_WIDTH) for k, x in flat.items()}
    return flat


def _inputs(case, placement):
    """flat NumPy inputs of the case, and the same values as the placement's ramba arrays"""
    import ramba_b200 as rb

    flat = flat_inputs(case, placement)
    if placement == "nd":
        arrays = {}
        for k, x in flat.items():
            w = onp.zeros((x.size // ND_WIDTH, ND_WIDTH + 5), dtype=x.dtype)
            w[:, :ND_WIDTH] = x.reshape(-1, ND_WIDTH)
            arrays[k] = rb.fromarray(w)[:, :ND_WIDTH]
        return flat, arrays
    return flat, {k: rb.fromarray(v) for k, v in flat.items()}


def evaluate(case, placement):
    """(outputs as flat NumPy arrays, [[plan, [[opcode, class, imm, stored view], ...], [view dtypes]], ...])"""
    import ramba_b200 as rb
    from ramba_b200 import _cabi
    from ramba_b200.runtime import RT

    flat, X = _inputs(case, placement)
    rb.sync()
    be = RT.be()
    run, plans = be.run, []
    cls_name = {0: "F64", 1: "F32", 2: "I64"}
    code_name = ["F64", "F32", "I64", "I32", "BOOL", "U8", "I8", "I16", "U16", "U32"]

    def record(fop, stream=None):
        insns = []
        for i in range(fop.n_insns):
            I = fop.insns[i]
            insns.append([_cabi.OPS[I.op], cls_name[I.ctype], int(I.imm), None if I.st_view == _cabi.NOSTORE else int(I.st_view)])
        plans.append([_cabi.describe_plan(fop), insns, [code_name[fop.views[v].dtype] for v in range(fop.n_views)]])
        return run(fop, stream)

    be.run = record
    try:
        outs = case.run(rb, X)
        rb.sync()
        got = [o.asarray().reshape(-1) for o in outs]
    finally:
        be.run = run
    return flat, got, plans


def _bits(x):
    x = onp.asarray(x)
    if x.dtype.kind == "f":
        u = x.view(onp.uint64 if x.dtype.itemsize == 8 else onp.uint32).copy()
        u[onp.isnan(x)] = 1  # NaN as NaN, whatever its payload and sign
        return u
    return x.astype(onp.int64) if x.dtype != onp.uint64 else x


def compare(case, flat, got):
    """mismatches of `got` against the case's expected values, bit for bit"""
    failures = []
    want = case.want(flat)
    assert len(want) == len(got), case.name
    for i, (w, g) in enumerate(zip(want, got)):
        if w.dtype == object:  # exact integers, wrapped to the dtype the engine gave the result
            w = onp.array([wrap(int(v), g.dtype) for v in w.tolist()], dtype=g.dtype)
        if w.dtype != g.dtype:
            failures.append("%s output %d: dtype %s, want %s" % (case.name, i, g.dtype, w.dtype))
            continue
        bad = _bits(w) != _bits(g)
        if bad.any():
            j = onp.flatnonzero(bad)
            seen, ex = set(), []
            for e in j:
                key = tuple(flat[k][e].item() for k in flat)
                if key not in seen:
                    seen.add(key)
                    ex.append("%s -> %r, want %r" % (key, g[e].item(), w[e].item()))
                if len(ex) == 6:
                    break
            failures.append("%s output %d: %d elements differ, e.g. %s" % (case.name, i, bad.sum(), "; ".join(ex)))
    return failures


def check_paths(case, placement, plans):
    """every op list ran on the kernel the placement is named for, and the case's ops and path were reached"""
    fails = []
    insns = [ins for _, ii, _ in plans for ins in ii]
    ops = {i[0] for i in insns}
    if not set(case.ops) <= ops:
        fails.append("%s [%s]: ops %s not in the op lists %s" % (case.name, placement, sorted(set(case.ops) - ops), sorted(ops)))
    # the op lists that do what the case is named for: its path, or else its opcodes
    mine = [(p, ii) for p, ii, views in plans if (case.check(p, ii, views) if case.check else set(case.ops) & {i[0] for i in ii})]
    if (case.check or case.ops) and not mine:
        fails.append("%s [%s]: the path it checks was not reached: %s" % (case.name, placement, plans))
    for plan, ii in mine:
        if not plan.startswith("kernel=general_interpreter form=elementwise "):
            continue
        want = " ndim=2 " if placement == "nd" else " ndim=1 "
        if want not in plan:
            fails.append("%s [%s]: %s" % (case.name, placement, plan))
    return fails


def _int_store_narrow(plan, insns, views):
    """an int64 view's values stored to a narrower integer view (not the fill of the fresh output)"""
    return "I64" in views and any(cls == "I64" and sv is not None and views[sv] not in ("I64", "F64", "F32") for op, cls, imm, sv in insns)


def _kernel(plan):
    if "variant=lean" in plan:
        return "lean"
    if plan.startswith("kernel=general_interpreter"):
        return "nd" if " ndim=1 " not in plan else ("generic" if "generic=" in plan else "1-D")
    return plan.split()[0][len("kernel="):]


# kernels (as _kernel names them) that the cases of a family must reach on a placement, in a process with default
# switches; "generic": a 1-D op list with instructions on the generic decode path.  The lean 1-D kernel takes the
# streaming kernel's vocabulary when that kernel is switched off (REACH_NO_STREAM).
REACH = {
    ("A", "1d"): {"1-D", "generic"}, ("A", "nd"): {"nd"},
    ("B", "1d"): {"1-D", "generic", "stream", "stream_terms"}, ("B", "nd"): {"nd", "stencil_tile", "stencil_terms"},
    ("C", "1d"): {"1-D", "generic", "stream_terms"}, ("C", "nd"): {"nd", "stencil_terms"},
}
REACH_NO_STREAM = {"lean", "1-D", "generic"}


def reach_failures(tag, kernels, want):
    seen = set().union(*kernels.values()) if kernels else set()
    return [] if want <= seen else ["%s: kernels %s never reached (reached: %s)" % (tag, sorted(want - seen), sorted(seen))]


def run_family(family, placement):
    failures, kernels = [], {}
    for case in cases():
        if case.family != family:
            continue
        flat, got, plans = evaluate(case, placement)
        failures += compare(case, flat, got)
        failures += check_paths(case, placement, plans)
        kernels[case.name] = sorted({_kernel(p) for p, _, _ in plans})
    return failures, kernels


def run_family_reaching(family, placement):
    failures, kernels = run_family(family, placement)
    return failures + reach_failures("%s %s" % (family, placement), kernels, REACH[family, placement]), kernels


# ---- D: library functions in ulps -------------------------------------------------------------------------------------
FUNCS = ["tan", "sinh", "cosh", "tanh", "asin", "acos", "atan", "exp", "log", "cbrt", "sqrt"]
MP = {"tan": mpmath.tan, "sinh": mpmath.sinh, "cosh": mpmath.cosh, "tanh": mpmath.tanh, "asin": mpmath.asin, "acos": mpmath.acos,
      "atan": mpmath.atan, "exp": mpmath.exp, "log": mpmath.log, "cbrt": mpmath.cbrt, "sqrt": mpmath.sqrt}
NP = {"asin": onp.arcsin, "acos": onp.arccos, "atan": onp.arctan}
RB = {"asin": "arcsin", "acos": "arccos", "atan": "arctan"}
SPECIALS = {  # compared bit for bit with NumPy's float64 results rounded to the class: exact at these arguments
    "tan": [0.0, -0.0, onp.inf, -onp.inf, onp.nan], "sinh": [0.0, -0.0, onp.inf, -onp.inf, onp.nan, 1000.0, -1000.0],
    "cosh": [0.0, -0.0, onp.inf, -onp.inf, onp.nan, 1000.0], "tanh": [0.0, -0.0, onp.inf, -onp.inf, onp.nan, 30.0, -30.0],
    "asin": [0.0, -0.0, 1.0, -1.0, 2.0, onp.nan], "acos": [1.0, 2.0, -2.0, onp.nan], "atan": [0.0, -0.0, onp.inf, -onp.inf, onp.nan],
    "exp": [0.0, -0.0, onp.inf, -onp.inf, onp.nan, 1000.0, -1000.0], "log": [0.0, -0.0, 1.0, -1.0, onp.inf, -onp.inf, onp.nan],
    "cbrt": [0.0, -0.0, -8.0, 27.0, onp.inf, -onp.inf, onp.nan], "sqrt": [0.0, -0.0, -1.0, onp.inf, -onp.inf, onp.nan, 4.0],
    "pow": [],
}


@functools.lru_cache(None)
def library_arguments(fn, dtype):
    """seeded arguments of fn in dtype: uniform samples at several scales over the domain, arguments near overflow and
    underflow, near 1 for log and +-1 for asin / acos, tiny and subnormal ones; all finite with a finite exact result"""
    rng = onp.random.default_rng(20261018 + FUNCS.index(fn) * 7 + (dtype == "float32"))
    f32 = dtype == "float32"
    k = 300
    sub = [5e-324, 1e-310, 2.2250738585072014e-308, 1e-300] if not f32 else [1.4e-45, 1e-40, 1.1754944e-38, 1e-30]
    tiny = sub + [1e-20, 1e-9]
    near1 = 1.0 + onp.arange(-20, 21) * (2.0 ** -52 if not f32 else 2.0 ** -23)
    lim = {"exp": ([709.78, 709.7, 700.0, -708.3, -745.13, -740.0, -744.0], [88.72, 88.0, -87.3, -103.9, -100.0, -95.0]),
           "sinh": ([710.47, 710.0, -710.47], [89.41, 89.0, -89.41]), "cosh": ([710.47, 710.0, -710.47], [89.41, 89.0, -89.41])}
    if fn in ("asin", "acos"):
        xs = [rng.uniform(-1, 1, k), rng.uniform(-1e-3, 1e-3, k), near1[near1 <= 1], -near1[near1 <= 1], tiny]
    elif fn in ("log", "sqrt"):
        xs = [rng.uniform(0, 10, k), onp.exp(rng.uniform(-690, 690, k)) if not f32 else onp.exp(rng.uniform(-87, 88, k)), near1, sub, [1e300 if not f32 else 3e38]]
    elif fn == "cbrt":
        xs = [rng.uniform(-10, 10, k), onp.exp(rng.uniform(-690, 690, k)) * rng.choice([-1, 1], k), sub, [-s for s in sub]]
    elif fn == "tan":
        xs = [rng.uniform(-1.6, 1.6, k), rng.uniform(-100, 100, k), rng.uniform(-1e5, 1e5, k), tiny]
    elif fn == "atan":
        xs = [rng.uniform(-1, 1, k), rng.uniform(-1e3, 1e3, k), onp.exp(rng.uniform(-40, 40, k)), tiny, [-t for t in tiny]]
    else:
        top = 709.0 if fn == "exp" else 710.0
        top = 88.0 if f32 and fn == "exp" else 89.0 if f32 else top
        xs = [rng.uniform(-1, 1, k), rng.uniform(-20, 20, k), rng.uniform(-top, top, k), tiny, [-t for t in tiny]]
        if fn in lim:
            xs.append(lim[fn][1 if f32 else 0])
    with onp.errstate(over="ignore"):
        x = onp.concatenate([onp.asarray(v, dtype=onp.float64) for v in xs]).astype(dtype)
    return onp.unique(x[onp.isfinite(x)])


@functools.lru_cache(None)
def pow_arguments(dtype):
    rng = onp.random.default_rng(20261019 + (dtype == "float32"))
    k = 600
    x = onp.concatenate([rng.uniform(0, 10, k), onp.exp(rng.uniform(-20, 20, k)), rng.uniform(0.9, 1.1, k), -rng.integers(1, 20, 50).astype(float)])
    y = onp.concatenate([rng.uniform(-30, 30, k), rng.uniform(-10, 10, k), rng.uniform(-500, 500, k), rng.integers(-20, 20, 50).astype(float) + 0.0])
    if dtype == "float32":
        y = onp.concatenate([rng.uniform(-30, 30, k), rng.uniform(-3, 3, k), rng.uniform(-200, 200, k), rng.integers(-10, 10, 50).astype(float)])
    return x.astype(dtype), y.astype(dtype)


def _dd(v):
    hi = libmp.to_float(v, rnd=libmp.round_nearest)
    if not math.isfinite(hi):
        return hi, 0.0
    return hi, libmp.to_float(libmp.mpf_sub(v, libmp.from_float(hi), PREC), rnd=libmp.round_nearest)


@functools.lru_cache(None)
def library_reference(fn, dtype):
    """(arguments, exact result rounded to float64, the remainder) for every argument of fn in dtype"""
    if fn == "pow":
        x, y = pow_arguments(dtype)
        with mpmath.workprec(PREC):
            ref = [_dd(mpmath.power(mpmath.mpf(float(p)), mpmath.mpf(float(q)))._mpf_) for p, q in zip(x, y)]
        args = (x, y)
    else:
        x = library_arguments(fn, dtype)
        with mpmath.workprec(PREC):
            ref = [_dd((MP[fn](mpmath.mpf(float(p))) if fn != "cbrt" else mpmath.sign(p) * mpmath.cbrt(abs(mpmath.mpf(float(p)))))._mpf_) for p in x]
        args = (x,)
    r = onp.array(ref, dtype=onp.float64).reshape(-1, 2)
    return args, r[:, 0], r[:, 1]


LIB_FORMS = ("float64", "float32", "float32 in float64")


def run_library(placement, forms=LIB_FORMS, floor=0.0):
    """{(fn, form): worst ulp error}, and the failures: results over their bound, specials that differ in any bit"""
    import ramba_b200 as rb

    failures, worst, kernels = [], {}, set()
    for fn in FUNCS + ["pow"]:
        for form in forms:
            dt = "float64" if form == "float64" else "float32"
            args, hi, lo = library_reference(fn, dt)
            n = args[0].size
            spec = onp.array(SPECIALS[fn], dtype=onp.float64).astype(dt)
            inputs = {"a": (list(args[0]) + list(spec), onp.dtype(dt).type)}
            if fn == "pow":
                inputs["b"] = (list(args[1]), onp.dtype(dt).type)

            def run(rb, X, fn=fn, form=form):
                a = X["a"] * 1.0 if form == "float32 in float64" else X["a"]
                if fn == "pow":
                    return [a ** X["b"]]
                return [getattr(rb, RB.get(fn, fn))(a)]

            case = Case("D", "%s %s" % (fn, form), inputs, run, None, (fn.upper(),))
            flat, got, plans = library_placed(case, placement)
            kernels |= {_kernel(p) for p, _, _ in plans}
            failures += check_paths(case, placement, plans)
            f, w = library_check(fn, form, got[0], flat, floor if form == "float64" else 0.0)
            failures += f
            if w is not None:
                worst[fn, form] = w
    return failures, worst, kernels


def library_bound(fn, form):
    """{form: ulp bound} of fn as this file holds it: the documented bound, or the recorded finding above it"""
    dt = "float64" if form == "float64" else "float32"
    b = ULP_BOUND[dt][fn]
    return FINDINGS.get((fn, form), 0.5 if b == 0 else float(b))


def library_check(fn, form, g, flat, floor=0.0):
    """(failures, worst ulp error) of the results g of fn in `form` at the arguments flat["a"] (and flat["b"]): each
    argument row (flat["row"]) below the reference count within its bound, the specials after them bit for bit"""
    dt = "float64" if form == "float64" else "float32"
    args, hi, lo = library_reference(fn, dt)
    n = args[0].size
    name = "%s %s" % (fn, form)
    if g.dtype != onp.dtype(dt):
        return ["%s: dtype %s" % (name, g.dtype)], None
    failures = []
    row = flat["row"]
    m = row < n
    gv = g[m].astype(onp.float64)
    h, l = hi[row[m]], lo[row[m]]
    err = ulp_error(gv, h, l) if form == "float64" else ulp_error(gv, h, l, onp.float32)
    with onp.errstate(invalid="ignore", over="ignore"):
        rounded = h.astype(dt)
    exact = ~onp.isfinite(rounded)  # overflow: the result must be the infinity
    e = onp.where(exact, 0.0, err)
    bound = rounded_bound(h) if form == "float32 in float64" else onp.full(h.size, max(floor, library_bound(fn, form)))
    worst = float(onp.nan_to_num(e, nan=onp.inf).max()) if e.size else 0.0
    bad = ~(e <= bound) | (exact & (_bits(g[m]) != _bits(rounded)))
    if bad.any():
        j = onp.flatnonzero(bad)[:5]
        failures.append("%s: %d over %s ulp, e.g. x=%r got=%r err=%r" % (name, bad.sum(), float(bound.max()), flat["a"][m][j].tolist(), gv[j].tolist(), e[j].tolist()))
    s = ~m
    if s.any():
        with onp.errstate(all="ignore"):
            sx = flat["a"][s]
            want = NP.get(fn, getattr(onp, fn, None))(sx.astype(onp.float64)).astype(dt)  # (NumPy's float32 cbrt(27) is 3 - 1 ulp)
        diff = _bits(want) != _bits(g[s])
        if diff.any():
            j = onp.flatnonzero(diff)[:6]
            failures.append("%s specials: x=%r got=%r want=%r" % (name, sx[j].tolist(), g[s][j].tolist(), want[j].tolist()))
    return failures, worst


def library_placed(case, placement):
    """the library case with its arguments laid out contiguously (plus a ragged tile), and each element's argument row"""
    import ramba_b200 as rb

    names = list(case.inputs)
    m = len(case.inputs["a"][0])
    size = -(-m // TILE) * TILE + RAGGED
    row = onp.arange(size) % m
    if "b" in case.inputs:
        nb = len(case.inputs["b"][0])
        row = onp.arange(size) % nb
    flat = {k: onp.asarray(case.inputs[k][0], dtype=case.inputs[k][1])[row] for k in names}
    if placement == "nd":
        rows = -(-size // ND_WIDTH)
        row = onp.resize(row, rows * ND_WIDTH)
        X = {}
        for k in names:
            x = onp.asarray(case.inputs[k][0], dtype=case.inputs[k][1])[row]
            flat[k] = x
            w = onp.zeros((rows, ND_WIDTH + 5), dtype=x.dtype)
            w[:, :ND_WIDTH] = x.reshape(rows, ND_WIDTH)
            X[k] = rb.fromarray(w)[:, :ND_WIDTH]
    else:
        X = {k: rb.fromarray(v) for k, v in flat.items()}
    c2 = Case(case.family, case.name, case.inputs, lambda rb, _X: case.run(rb, X), None, case.ops)
    c2.inputs = {names[0]: ([0.0], onp.float64)}  # evaluate() lays out a dummy; the real operands are X
    _, got, plans = evaluate(c2, "1d")
    flat["row"] = row
    return flat, got, plans


# ---- CPU --------------------------------------------------------------------------------------------------------------
def _exact(case, flat):
    """the case's expected outputs in their final dtypes (exact integers wrapped to the dtype they are declared in)"""
    out = []
    for w in case.want(flat):
        out.append(onp.array([int(v) for v in w.tolist()], dtype=onp.int64) if w.dtype == object else onp.asarray(w))
    return out


def _ftz(x):
    x = onp.array(x, copy=True)
    x[(x != 0) & (onp.abs(x) < onp.finfo(x.dtype).tiny)] = 0
    return x


def _saturate(x, lo, hi):
    with onp.errstate(invalid="ignore"):
        return onp.where(onp.isnan(x), 0, onp.clip(onp.trunc(onp.nan_to_num(x, posinf=hi, neginf=lo)), lo, hi))


WRONG = {  # case -> a plausible wrong restatement of it, from the flat inputs
    "float64 //": lambda x: [onp.where(x["b"] == 0, onp.nan, onp.floor_divide(x["a"], x["b"]))],   # no zero-divisor branch
    "float32 //": lambda x: [onp.where(x["b"] == 0, onp.float32(onp.nan), onp.floor_divide(x["a"], x["b"]))],
    "float64 * 1 stored to int64": lambda x: [_saturate(x["a"], -2.0 ** 63, 2.0 ** 63 - 1024).astype(onp.int64)],  # cvt.rzi
    "float32 * 1 stored to int32": lambda x: [_saturate(x["a"].astype(onp.float64), -2.0 ** 31, 2.0 ** 31 - 1).astype(onp.int32)],  # straight to int32
    "float64 astype int32, + 1": lambda x: [_saturate(x["a"], -2.0 ** 31, 2.0 ** 31 - 1).astype(onp.int32),
                                            _saturate(x["a"], -2.0 ** 31, 2.0 ** 31 - 1).astype(onp.int64) + 1],
    "float64 masked into a dead int64 temporary, + 1": lambda x: [onp.where(x["m"], _saturate(x["a"], -2.0 ** 63, 2.0 ** 63 - 1024).astype(onp.int64),
                                                                            2 * x["i"]) + 1],
    "float64 subnormals": None,  # every output flushed to zero: built from the right outputs below
    "float32 subnormals": None,
    "float64 minimum": lambda x: [_elementwise(lambda p, q: py_min(q, p), x["a"], x["b"], out=onp.float64)],  # operands swapped
    "float32 maximum": lambda x: [_elementwise(lambda p, q: py_max(q, p), x["a"], x["b"], out=onp.float32)],
    "int64 <<": lambda x: [_elementwise(lambda p, q: wrap(p << (q & 63)), x["a"], x["b"])],  # count masked with & 63
    "int64 >>": lambda x: [_elementwise(lambda p, q: p >> (q & 63), x["a"], x["b"])],
}


def test_the_rules_fail_on_wrong_restatements():
    """compare() passes each case's exact outputs and rejects a plausible wrong restatement of it; library_check passes
    the correctly rounded results of every function and form and rejects them moved away by more than the bound"""
    by_name = {c.name: c for c in cases()}
    assert set(WRONG) <= set(by_name)
    for name, wrong in WRONG.items():
        case = by_name[name]
        flat = flat_inputs(case, "1d")
        right = _exact(case, flat)
        assert compare(case, flat, right) == [], name
        bad = [_ftz(w) for w in right] if wrong is None else wrong(flat)
        assert compare(case, flat, bad), name
    for fn in FUNCS + ["pow"]:
        for form in LIB_FORMS:
            dt = "float64" if form == "float64" else "float32"
            args, hi, lo = library_reference(fn, dt)
            spec = onp.array(SPECIALS[fn], dtype=onp.float64)
            flat = {"a": onp.concatenate([args[0], spec.astype(dt)]), "row": onp.arange(args[0].size + spec.size)}
            with onp.errstate(all="ignore"):
                good = onp.concatenate([hi.astype(dt)] + ([NP.get(fn, getattr(onp, fn, None))(spec).astype(dt)] if spec.size else []))
            assert library_check(fn, form, good, flat)[0] == [], (fn, form)
            steps = max(3, int(library_bound(fn, form)) + 1)  # a function 3 ulp off, or one ulp past a wider bound
            off = good.copy()
            for _ in range(steps):
                off[: args[0].size] = onp.nextafter(off[: args[0].size], onp.copysign(onp.inf, off[: args[0].size]))
            assert library_check(fn, form, off, flat)[0], (fn, form)
            flipped = good.copy()
            flipped[args[0].size:] = -flipped[args[0].size:]  # specials with the wrong sign
            if (_bits(flipped) != _bits(good)).any():
                assert library_check(fn, form, flipped, flat)[0], (fn, form)
    # the independent rules themselves at the points the issue names
    assert f2i(onp.inf) == I64_MIN and f2i(onp.nan) == I64_MIN and wrap(f2i(3e9), onp.int32) == -1294967296
    assert int_power(2, 64) == 0 and int_power(-1, -3) == -1 and int_power(0, -1) == 0
    assert to_f32_once((1 << 60) + (1 << 36) + 1) == onp.float32(2.0 ** 60 + 2.0 ** 37) != onp.float32(float((1 << 60) + (1 << 36) + 1))


def test_the_layout_puts_every_value_at_every_position():
    cols, row = spread([list(range(9))])
    e = onp.arange(row.size)
    for i in range(9):
        pos = e[row == i]
        assert set((pos % TILE) // 256) == set(range(8)) and set(pos % 256) == set(range(256))
    assert row.size % TILE == RAGGED


@pytest.mark.parametrize("family", ["A", "B", "C"])
@pytest.mark.parametrize("placement", ["1d", "nd"])
def test_exact_families_on_the_oracle(oracle_engine, family, placement):
    failures, _ = run_family_reaching(family, placement)
    assert not failures, "\n".join(failures)


def test_library_functions_on_the_oracle(oracle_engine):
    """glibc's float64 functions behind the oracle within CUDA's bounds or 2 ulp, whichever is wider (glibc's tanh
    reaches 1.11 ulp on these arguments), specials bit for bit; NumPy's own float32 routines are not held to CUDA's
    float32 bounds"""
    failures, worst, _ = run_library("1d", ("float64", "float32 in float64"), floor=2.0)
    assert not failures, "\n".join(failures)


def test_full_kernel_placement_plans(tmp_path):
    out = _run_switched(tmp_path, "RB200_NO_LEAN_INTERP", "plans")
    assert not out["failures"], "\n".join(out["failures"])


def test_lean_kernel_placement_plans(tmp_path):
    out = _run_switched(tmp_path, "RB200_NO_STREAM_KERNEL", "plans")
    assert not out["failures"], "\n".join(out["failures"])


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _report(tag, worst=None, kernels=None):
    if kernels:
        print("kernels, %s: %s" % (tag, json.dumps(kernels, sort_keys=True)))
    if worst:
        print("worst ulp, %s: %s" % (tag, ", ".join("%s %s %.3f" % (f, k, u) for (f, k), u in sorted(worst.items()))))


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["A", "B", "C"])
@pytest.mark.parametrize("placement", ["1d", "nd"])
def test_exact_families(gpu_engine, family, placement):
    failures, kernels = run_family_reaching(family, placement)
    _report("%s %s" % (family, placement), kernels=kernels)
    assert not failures, "\n".join(failures)


@pytest.mark.gpu
@pytest.mark.parametrize("placement", ["1d", "nd"])
def test_library_functions(gpu_engine, placement):
    failures, worst, kernels = run_library(placement)
    _report(placement, worst, sorted(kernels))
    failures += reach_failures("library %s" % placement, {"all": kernels}, {"nd"} if placement == "nd" else {"generic"})
    assert not failures, "\n".join(failures)


def _switched_worker(out_dir, mode):
    """Families A-C on the 1-D placement in a process whose kill switch is set (read once per process):
    RB200_NO_LEAN_INTERP keeps every op list off the lean kernel, RB200_NO_STREAM_KERNEL hands the streaming kernel's
    vocabulary (neg, abs, min, max, f32 <-> f64) to the lean kernel"""
    from ramba_b200.runtime import RT

    RT.reset()
    if mode == "plans":
        import _oracle_backend

        _oracle_backend.install()
    elif os.environ.get("RB200_DRY_GPU_TESTS"):
        import conftest

        conftest._dry_gpu()
    failures, kernels = [], {}
    for fam in ("A", "B", "C"):
        f, k = run_family(fam, "1d")
        failures += f
        kernels.update(k)
    seen = set().union(*kernels.values())
    if os.environ.get("RB200_NO_LEAN_INTERP") and "lean" in seen:
        failures.append("RB200_NO_LEAN_INTERP: an op list ran on the lean kernel")
    if os.environ.get("RB200_NO_STREAM_KERNEL"):
        failures += reach_failures("RB200_NO_STREAM_KERNEL", kernels, REACH_NO_STREAM)
        if seen & {"stream", "stream_terms"}:
            failures.append("RB200_NO_STREAM_KERNEL: an op list ran on the streaming kernel")
    with open(os.path.join(out_dir, "out.json"), "w") as fh:
        json.dump({"failures": failures, "kernels": kernels}, fh)


def _run_switched(tmp_path, switch, mode):
    code = "import sys; sys.path[:0] = [%r, %r]; import test_elementwise_semantics as t; t._switched_worker(%r, %r)" % (ROOT, HERE, str(tmp_path), mode)
    env = dict(os.environ, **{switch: "1"})
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    with open(os.path.join(str(tmp_path), "out.json")) as f:
        return json.load(f)


def _switched_on_gpu(tmp_path, switch):
    out = _run_switched(tmp_path, switch, "gpu")
    _report("1d, " + switch, kernels=out["kernels"])
    assert not out["failures"], "\n".join(out["failures"])


@pytest.mark.gpu
def test_exact_families_off_the_lean_kernel(gpu_engine, tmp_path):
    _switched_on_gpu(tmp_path, "RB200_NO_LEAN_INTERP")


@pytest.mark.gpu
def test_exact_families_off_the_stream_kernel(gpu_engine, tmp_path):
    _switched_on_gpu(tmp_path, "RB200_NO_STREAM_KERNEL")
