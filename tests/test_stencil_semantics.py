"""The shifted-view stencil kernels (stencil_tile_kernel and stencil_terms_kernel in rb200_tile.cu) held to per-operation
NumPy references, bit for bit, on every plan they reach.

Every expected value is a NumPy expression written in the case itself with explicit dtypes (Numba's typing: float32 op
float32 rounds in float32, float32 op a Python float or float64 is float64, the store converts; one rounding per
operation, the order of the statement).  The oracle, the op list and the fuser never compute an expected value.  Each
case also states the opcodes and classes of its op list (so a wrong typing assumption fails loudly) and the plan fields
that rb200_describe_plan must report for it: kernel, loader, element size, term split, fast tail, ring depth, halo,
z-chunking and TMA corner shift.  Inputs carry NaN, +-inf, -0.0 and subnormals at tile, halo and z-chunk edges.

  * CPU: every case on the oracle backend, with its plan (the planner runs on the host), in one process per set of
    kernel switches; gloo worlds of 2, 3, 4 and 8 ranks with splits along every axis; and every check shown to reject a
    wrong restatement (float32 phase done in float64, a dropped term, a halo off by one, a contracted multiply-add, a
    border overwritten by sstencil).
  * GPU: the same cases on the H100 under the default switches, RB200_NO_TERMS_KERNEL, RB200_NO_TMA and
    RB200_NO_TILE_KERNEL (one process each: the switches are read once per process), and one float32 Laplacian of more
    than 2^31 elements checked on sampled planes."""
import json
import os
import socket
import subprocess
import sys

import numpy as onp
import pytest

from _stencil_ref import F32, F64, edge_data, fma64, mismatches

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def c64(x):
    return onp.asarray(x).astype(F64)


def _cls(dt):
    return "F32" if dt == F32 else "F64"


class Case:
    """inputs: {name: host array}; run(np, X) -> outputs (np: the ramba module, X: the inputs as ramba arrays);
    want(x) -> expected host arrays; ops: the op list's instructions as 'OP.CLASS' (one op list of the run must be exactly
    this); plan: {describe_plan field: value} for that op list under the default switches"""

    def __init__(self, name, inputs, run, want, ops, plan=None, border=None):
        self.name, self.inputs, self.run, self.want, self.ops, self.plan = name, inputs, run, want, ops, plan or {}
        self.border = border  # {"local_border": k} for padded shards


CASES = []


def case(*a, **k):
    CASES.append(Case(*a, **k))


# ---- 3-D Laplacian: the BASELINE program ------------------------------------------------------------------------------
def lap_want(u, dt, out=None):
    a, b = u[:-2, 1:-1, 1:-1], u[2:, 1:-1, 1:-1]
    c, d = u[1:-1, :-2, 1:-1], u[1:-1, 2:, 1:-1]
    e, f, m = u[1:-1, 1:-1, :-2], u[1:-1, 1:-1, 2:], u[1:-1, 1:-1, 1:-1]
    s = ((((a + b) + c) + d) + e) + f  # in the data's class
    v = onp.zeros(u.shape, dt) if out is None else out
    v[1:-1, 1:-1, 1:-1] = (c64(s) - 6.0 * c64(m)).astype(dt)
    return [v]


def lap_run(np, X):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    V[1:-1, 1:-1, 1:-1] = (U[:-2, 1:-1, 1:-1] + U[2:, 1:-1, 1:-1] + U[1:-1, :-2, 1:-1] + U[1:-1, 2:, 1:-1]
                           + U[1:-1, 1:-1, :-2] + U[1:-1, 1:-1, 2:] - 6.0 * U[1:-1, 1:-1, 1:-1])
    return [V]


LAP_OPS = {F32: ["ADD.F32"] * 5 + ["CVT.F64", "MULSUB.F64"], F64: ["ADD.F64"] * 5 + ["MULSUB.F64"]}

# interior boxes (Z, Y, X): X in {1, 2, 127, 128, 129, 143, 144, 145, 257}, Y in {1, 15, 16, 17}, Z in {1, 2, 15, 16, 17}
for i, (z, y, x) in enumerate([(1, 1, 1), (2, 15, 2), (15, 16, 127), (16, 17, 128), (17, 1, 129), (2, 16, 143),
                               (16, 15, 144), (15, 17, 145), (17, 16, 257)]):
    for dt in (F32, F64):
        if dt == F64 and i % 2:
            continue
        # (a 1 x 1 x 1 box collapses to 1-D and leaves the stencil kernels)
        k = "stencil_terms" if i else ("stream_terms" if dt == F32 else "general_interpreter")
        case("lap_%dx%dx%d_%s" % (z, y, x, dt.__name__), {"u": edge_data((z + 2, y + 2, x + 2), dt, 100 + i)}, lap_run,
             lambda x, dt=dt: lap_want(x["u"], dt), LAP_OPS[dt], {"kernel": k})
# TMA rows (132 floats, 130 doubles) and the term split: f32 runs six terms in float32 and one weighted tail in float64
case("lap_tma_f32", {"u": edge_data((20, 36, 132), F32, 1)}, lap_run, lambda x: lap_want(x["u"], F32), LAP_OPS[F32],
     {"kernel": "stencil_terms", "elem": "4", "loader": "tma", "terms": "7(f32:6)", "fast_tail": "1", "ring": "5",
      "halo": "z0+2,y1+1,x1+1", "corner_shift": "0"})
case("lap_tma_f64", {"u": edge_data((12, 40, 130), F64, 2)}, lap_run, lambda x: lap_want(x["u"], F64), LAP_OPS[F64],
     {"kernel": "stencil_terms", "elem": "8", "loader": "tma", "terms": "7(f32:0)", "fast_tail": "0", "ring": "4"})
case("lap_odd_f32", {"u": edge_data((9, 35, 131), F32, 3)}, lap_run, lambda x: lap_want(x["u"], F32), LAP_OPS[F32],
     {"kernel": "stencil_terms", "loader": "cp.async"})
# a source that is an offset view of a larger array, and one with padded shards
case("lap_offset_view_f32", {"big": edge_data((23, 39, 140), F32, 4)},
     lambda np, X: lap_run(np, {"u": X["big"][3:, 2:, 5:]}), lambda x: lap_want(x["big"][3:, 2:, 5:], F32), LAP_OPS[F32],
     {"kernel": "stencil_terms"})
case("lap_local_border_f64", {"u": edge_data((14, 33, 150), F64, 5)}, lap_run, lambda x: lap_want(x["u"], F64),
     LAP_OPS[F64], {"kernel": "stencil_terms"}, border={"local_border": 2})
# -0.0 neighbour sums stay -0.0 (the Laplacian's -6.0 * -0.0 tail makes +0.0: -0.0 - -0.0)
for dt in (F32, F64):
    case("negzero_sum_%s" % dt.__name__, {"u": onp.full((6, 20, 140), -0.0, dt)},
         lambda np, X: _sum4(np, X["u"]), lambda x, dt=dt: _sum4_want(x["u"], dt), ["ADD.%s" % _cls(dt)] * 3,
         {"kernel": "stencil_terms", "terms": "4(f32:%d)" % (4 if dt == F32 else 0)})


def _sum4(np, U):
    V = np.zeros(U.shape, dtype=U.dtype)
    V[1:-1, 1:-1, 1:-1] = U[1:-1, :-2, 1:-1] + U[1:-1, 2:, 1:-1] + U[1:-1, 1:-1, :-2] + U[1:-1, 1:-1, 2:]
    return [V]


def _sum4_want(u, dt):
    v = onp.zeros(u.shape, dt)
    v[1:-1, 1:-1, 1:-1] = ((u[1:-1, :-2, 1:-1] + u[1:-1, 2:, 1:-1]) + u[1:-1, 1:-1, :-2]) + u[1:-1, 1:-1, 2:]
    return [v]


# ---- 2-D Laplacian over the same size sweep: X in {1, 2, 127, 128, 129, 143, 144, 145, 257}, Y in {1, 15, 16, 17}.  Rows
# shorter than 64 elements have no staged group; a box of one row or one column collapses to 1-D (streaming kernel).
def lap2_want(u, dt):
    s = ((u[:-2, 1:-1] + u[2:, 1:-1]) + u[1:-1, :-2]) + u[1:-1, 2:]  # in the data's class
    v = onp.zeros(u.shape, dt)
    v[1:-1, 1:-1] = (c64(s) - 4.0 * c64(u[1:-1, 1:-1])).astype(dt)
    return [v]


def lap2_run(np, X):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    V[1:-1, 1:-1] = U[:-2, 1:-1] + U[2:, 1:-1] + U[1:-1, :-2] + U[1:-1, 2:] - 4.0 * U[1:-1, 1:-1]
    return [V]


LAP2_OPS = {F32: ["ADD.F32"] * 3 + ["CVT.F64", "MULSUB.F64"], F64: ["ADD.F64"] * 3 + ["MULSUB.F64"]}
for i, (y, x) in enumerate([(1, 1), (15, 2), (16, 127), (17, 128), (1, 129), (16, 143), (15, 144), (17, 145), (16, 257),
                            (17, 1)]):
    for dt in (F32, F64):
        k = "stencil_terms" if y > 1 and x > 1 else "stream_terms"
        case("lap2d_%dx%d_%s" % (y, x, dt.__name__), {"u": edge_data((y + 2, x + 2), dt, 200 + i)}, lap2_run,
             lambda x, dt=dt: lap2_want(x["u"], dt), LAP2_OPS[dt], {"kernel": k})


# ---- z halos of 1, 2 and 3 on a persistent grid with more items than CTAs (Z = 16 k + 1: the last chunk is short) --------
def zhalo_run(np, X, hz):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    V[hz:, 1:-1, 1:-1] = U[hz:, 1:-1, 1:-1] + U[:-hz, 1:-1, 1:-1] + U[hz:, :-2, 1:-1] - 0.25 * U[hz:, 2:, 1:-1]
    return [V]


def zhalo_want(u, hz):
    v = onp.zeros(u.shape, F32)
    s = (u[hz:, 1:-1, 1:-1] + u[:-hz, 1:-1, 1:-1]) + u[hz:, :-2, 1:-1]
    v[hz:, 1:-1, 1:-1] = (c64(s) - 0.25 * c64(u[hz:, 2:, 1:-1])).astype(F32)
    return [v]


for hz in (1, 2, 3):
    case("zhalo%d_items_f32" % hz, {"u": edge_data((1073 + hz, 19, 259), F32, 10 + hz)},
         lambda np, X, hz=hz: zhalo_run(np, X, hz), lambda x, hz=hz: zhalo_want(x["u"], hz),
         ["ADD.F32", "ADD.F32", "CVT.F64", "MULSUB.F64"],
         {"kernel": "stencil_terms", "halo": "z%d+0,y1+1,x0+0" % hz, "planes_per_item": "16", "terms": "4(f32:3)",
          "fast_tail": "1", "items": "408", "ctas": "396", "ring": str(hz + 3)})


# ---- halo shifts at the group limits: dy / dx of +-8 stay in the group, +-9 make a direct view --------------------------
M = 9


def sh2(u, dy, dx):
    n, m = u.shape
    return u[M + dy:n - M + dy, M + dx:m - M + dx]


def shifts_run(np, X, shifts):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    acc = sh2(U, 0, 0)
    for dy, dx in shifts:
        acc = acc + sh2(U, dy, dx)
    V[M:-M, M:-M] = acc
    return [V]


def shifts_want(u, shifts):
    v = onp.zeros(u.shape, u.dtype)
    acc = sh2(u, 0, 0)
    for dy, dx in shifts:
        acc = acc + sh2(u, dy, dx)  # float32 + float32 in float32
    v[M:-M, M:-M] = acc
    return [v]


for tag, shifts, staged in [("dy+8", [(8, 0)], 2), ("dy-8", [(-8, 0)], 2), ("dy+9", [(9, 0), (-1, 0)], 2),
                            ("dy-9", [(-9, 0), (1, 0)], 2), ("dx+8", [(0, 8)], 2), ("dx-8", [(0, -8)], 2),
                            ("dx+9", [(0, 9), (0, -1)], 2), ("dx-9", [(0, -9), (0, 1)], 2),
                            ("xspan16", [(0, -8), (0, 8)], 3)]:
    n_terms = len(shifts) + 1
    case("halo_%s_f32" % tag, {"u": edge_data((60, 300), F32, 20)}, lambda np, X, s=shifts: shifts_run(np, X, s),
         lambda x, s=shifts: shifts_want(x["u"], s), ["ADD.F32"] * len(shifts),
         {"kernel": "stencil_terms", "staged_views": str(staged), "terms": "%d(f32:%d)" % (n_terms, n_terms)})


# ---- dz span 3 (in the group) and 4 (beyond the ring) -------------------------------------------------------------------
def zspan_run(np, X, dzs):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    acc = U[4:-4, 1:-1, 1:-1]
    for dz in dzs:
        acc = acc + U[4 + dz:U.shape[0] - 4 + dz, 1:-1, 1:-1]
    V[4:-4, 1:-1, 1:-1] = acc
    return [V]


def zspan_want(u, dzs):
    v = onp.zeros(u.shape, u.dtype)
    acc = u[4:-4, 1:-1, 1:-1]
    for dz in dzs:
        acc = acc + u[4 + dz:u.shape[0] - 4 + dz, 1:-1, 1:-1]
    v[4:-4, 1:-1, 1:-1] = acc
    return [v]


for tag, dzs, plan in [("3", [3], {"kernel": "stencil_terms", "halo": "z0+3,y0+0,x0+0", "staged_views": "2"}),
                       ("-3", [-3], {"kernel": "stencil_terms", "halo": "z3+0,y0+0,x0+0"}),
                       ("4", [4, -1], {"kernel": "stencil_terms", "halo": "z1+0,y0+0,x0+0", "staged_views": "2"}),
                       # three members spanning four planes: more than the ring holds, the tile kernel declines
                       ("-2+2", [-2, 2], {"kernel": "general_interpreter"})]:
    case("zspan%s_f64" % tag, {"u": edge_data((30, 20, 140), F64, 21)}, lambda np, X, d=dzs: zspan_run(np, X, d),
         lambda x, d=dzs: zspan_want(x["u"], d), ["ADD.F64"] * len(dzs), plan)


# ---- row strides of 63 and 64 (64: the smallest row stride of a staged group) ---------------------------------------------
def sum4_2d_run(np, X):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    V[1:-1, 1:-1] = U[:-2, 1:-1] + U[2:, 1:-1] + U[1:-1, :-2] + U[1:-1, 2:]
    return [V]


def sum4_2d_want(u):
    v = onp.zeros(u.shape, u.dtype)
    v[1:-1, 1:-1] = ((u[:-2, 1:-1] + u[2:, 1:-1]) + u[1:-1, :-2]) + u[1:-1, 2:]
    return [v]


case("rowstride63_f32", {"u": edge_data((40, 63), F32, 30)}, sum4_2d_run, lambda x: sum4_2d_want(x["u"]), ["ADD.F32"] * 3,
     {"kernel": "stencil_terms", "loader": "none", "staged_views": "0", "direct_views": "5"})
case("rowstride64_f32", {"u": edge_data((40, 64), F32, 31)}, sum4_2d_run, lambda x: sum4_2d_want(x["u"]), ["ADD.F32"] * 3,
     {"kernel": "stencil_terms", "loader": "tma", "staged_views": "4"})


# ---- few rows per plane: a shift of two rows in planes of four rows decodes as (dz, dy) = (1, -2) -----------------------
def fewrows_run(np, X):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    V[1:-1, 1:3, 1:-1] = U[1:-1, 2:, 1:-1] + U[1:-1, :-2, 1:-1] + U[:-2, 1:3, 1:-1] + U[2:, 1:3, 1:-1]
    return [V]


def fewrows_want(u):
    v = onp.zeros(u.shape, u.dtype)
    v[1:-1, 1:3, 1:-1] = ((u[1:-1, 2:, 1:-1] + u[1:-1, :-2, 1:-1]) + u[:-2, 1:3, 1:-1]) + u[2:, 1:3, 1:-1]
    return [v]


for dt, x in ((F32, 132), (F64, 130)):
    case("fewrows_%s" % dt.__name__, {"u": edge_data((40, 4, x), dt, 32)}, fewrows_run, lambda x: fewrows_want(x["u"]),
         ["ADD.%s" % _cls(dt)] * 3, {"kernel": "stencil_terms", "staged_views": "4", "halo": "z1+1,y2+0,x0+0",
                                     "loader": "cp.async", "corner_shift": "1"})


# ---- a 16-byte aligned group whose halo'd box would start before its buffer: the first view is the group's reference,
# the second decodes as (dz, dy) = (1, -2), so the box corner lies two rows (264 floats) before the allocation.  The
# aligned corner and whole 16-byte rows would allow TMA; only the bounds check sends it to the predicated cp.async
# loader.  The same two views in the other order make the second one the reference and stay inside: TMA. --------------
def past_run(np, X, first_low):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    lo, hi = U[:, :-2, :128], U[:, 2:, :128]
    V[:, 2:, :128] = lo + hi if first_low else hi + lo
    return [V]


def past_want(u, first_low):
    v = onp.zeros(u.shape, u.dtype)
    lo, hi = u[:, :-2, :128], u[:, 2:, :128]
    v[:, 2:, :128] = lo + hi if first_low else hi + lo
    return [v]


for first_low, loader, halo in ((True, "cp.async", "z0+1,y2+0,x0+0"), (False, "tma", "z0+0,y2+0,x0+0")):
    case("box_%s_buffer_f32" % ("past" if first_low else "inside"), {"u": edge_data((30, 4, 132), F32, 33)},
         lambda np, X, f=first_low: past_run(np, X, f), lambda x, f=first_low: past_want(x["u"], f), ["ADD.F32"],
         {"kernel": "stencil_terms", "staged_views": "2", "halo": halo, "loader": loader, "corner_shift": "0"})


# ---- corners at every 16-byte misalignment: 0-3 elements (float32), 0-1 (float64).  Rows of 104 elements with the halo:
# whole 16-byte units, so only the corner decides the loader (TMA on a 16-byte boundary, cp.async past it) ----------------
def corner_run(np, X, c):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    V[1:-1, c + 1:c + 103] = U[:-2, c + 1:c + 103] + U[2:, c + 1:c + 103] + U[1:-1, c:c + 102] + U[1:-1, c + 2:c + 104]
    return [V]


def corner_want(u, c):
    v = onp.zeros(u.shape, u.dtype)
    v[1:-1, c + 1:c + 103] = ((u[:-2, c + 1:c + 103] + u[2:, c + 1:c + 103]) + u[1:-1, c:c + 102]) + u[1:-1, c + 2:c + 104]
    return [v]


for dt, m, shifts in ((F32, 132, (0, 1, 2, 3)), (F64, 130, (0, 1))):
    for c in shifts:
        case("corner%d_%s" % (c, dt.__name__), {"u": edge_data((50, m), dt, 40 + c)}, lambda np, X, c=c: corner_run(np, X, c),
             lambda x, c=c: corner_want(x["u"], c), ["ADD.%s" % _cls(dt)] * 3,
             {"kernel": "stencil_terms", "loader": "cp.async" if c else "tma", "corner_shift": str(c)})


# ---- direct operands: transposed, reversed, strided, broadcast ----------------------------------------------------------
def direct_run(np, X):
    U, T, R, S, b = X["u"], X["t"], X["r"], X["s"], X["b"]
    V = np.zeros(U.shape, dtype=U.dtype)
    V[1:-1, 1:-1] = (U[:-2, 1:-1] + U[2:, 1:-1] + T.T[1:-1, 1:-1] + R[::-1, ::-1][1:-1, 1:-1]
                     + S[2:-2:2, 2:-2:2] + b[1:-1])
    return [V]


def direct_want(x):
    u, t, r, s, b = x["u"], x["t"], x["r"], x["s"], x["b"]
    v = onp.zeros(u.shape, u.dtype)
    v[1:-1, 1:-1] = ((((u[:-2, 1:-1] + u[2:, 1:-1]) + t.T[1:-1, 1:-1]) + r[::-1, ::-1][1:-1, 1:-1]) + s[2:-2:2, 2:-2:2]) + b[None, 1:-1]
    return [v]


case("direct_kinds_f32", {"u": edge_data((70, 200), F32, 50), "t": edge_data((200, 70), F32, 51), "r": edge_data((70, 200), F32, 52),
                          "s": edge_data((140, 400), F32, 53), "b": edge_data((200,), F32, 54)}, direct_run, direct_want,
     ["ADD.F32"] * 5, {"kernel": "stencil_terms", "staged_views": "2", "direct_views": "5"})


# ---- term splits and the float32 phase ----------------------------------------------------------------------------------
def mixed_run(np, X):
    """BUG REPRODUCER: a float64 group behind a float32 prefix of direct views"""
    U, A, B = X["u"], X["a"], X["b"]
    V = np.zeros(U.shape)
    V[1:-1, 1:-1] = ((A[1:-1, 1:-1] + B[1:-1, 1:-1]) + U[:-2, 1:-1]) + U[2:, 1:-1]
    return [V]


def mixed_want(x):
    u, a, b = x["u"], x["a"], x["b"]
    v = onp.zeros(u.shape, F64)
    v[1:-1, 1:-1] = (c64(a[1:-1, 1:-1] + b[1:-1, 1:-1]) + u[:-2, 1:-1]) + u[2:, 1:-1]
    return [v]


def _overflowing(shape, seed):
    """float32 data whose pairwise float32 sums overflow at many places, and round differently from float64 elsewhere"""
    a = edge_data(shape, F32, seed)
    a.reshape(-1)[::7] = F32(3.0e38)
    return a


case("f32_prefix_f64_group", {"u": edge_data((70, 200), F64, 60), "a": _overflowing((70, 200), 61), "b": _overflowing((70, 200), 62)},
     mixed_run, mixed_want, ["ADD.F32", "CVT.F64", "ADD.F64", "ADD.F64"],
     {"kernel": "stencil_tile", "elem": "8", "staged_views": "2", "terms": "0(f32:0)", "chains": "1"})


def promote_run(np, X):
    U = X["u"]
    V = np.zeros(U.shape)  # float64 destination: the float32 phase's overflow and rounding show in the stored value
    V[1:-1, 1:-1] = (U[:-2, 1:-1] + U[2:, 1:-1]) - 0.5 * U[1:-1, 1:-1]
    return [V]


def promote_want(x):
    u = x["u"]
    v = onp.zeros(u.shape, F64)
    v[1:-1, 1:-1] = c64(u[:-2, 1:-1] + u[2:, 1:-1]) - 0.5 * c64(u[1:-1, 1:-1])
    return [v]


case("f32_overflow_before_promotion", {"u": _overflowing((70, 264), 63)}, promote_run, promote_want,
     ["ADD.F32", "CVT.F64", "MULSUB.F64"],
     {"kernel": "stencil_terms", "elem": "4", "terms": "3(f32:2)", "fast_tail": "1", "loader": "cp.async"})


def split_run(np, X):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    V[1:-1, 1:-1] = (U[:-2, 1:-1] + U[2:, 1:-1] + U[1:-1, :-2]) - 0.5 * U[1:-1, 2:] + 0.25 * U[1:-1, 1:-1]
    return [V]


def split_want(x):
    u = x["u"]
    v = onp.zeros(u.shape, F32)
    s = (u[:-2, 1:-1] + u[2:, 1:-1]) + u[1:-1, :-2]
    v[1:-1, 1:-1] = ((c64(s) - 0.5 * c64(u[1:-1, 2:])) + 0.25 * c64(u[1:-1, 1:-1])).astype(F32)
    return [v]


case("split_no_fast_tail_f32", {"u": edge_data((50, 270), F32, 64)}, split_run, split_want,
     ["ADD.F32", "ADD.F32", "CVT.F64", "MULSUB.F64", "MULADD.F64"],
     {"kernel": "stencil_terms", "terms": "5(f32:3)", "fast_tail": "0"})


def weighted_run(np, X):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    V[1:-1, 1:-1] = 0.3 * U[:-2, 1:-1] + 0.7 * U[2:, 1:-1] - 0.1 * U[1:-1, 1:-1]
    return [V]


def weighted_want(x):
    u = c64(x["u"])
    v = onp.zeros(u.shape, x["u"].dtype)
    v[1:-1, 1:-1] = ((0.3 * u[:-2, 1:-1] + 0.7 * u[2:, 1:-1]) - 0.1 * u[1:-1, 1:-1]).astype(x["u"].dtype)
    return [v]


for dt in (F32, F64):  # float32 data in the float64 class from the first term: f32:0 at elem 4
    case("weighted_%s" % dt.__name__, {"u": edge_data((50, 270), dt, 65)}, weighted_run, weighted_want,
         ["MUL.F64", "MULADD.F64", "MULSUB.F64"], {"kernel": "stencil_terms", "terms": "4(f32:0)", "elem": "4" if dt == F32 else "8"})


# ---- the lean-machine form: registers, chains, ops outside the term vocabulary ---------------------------------------------
def regs_run(np, X):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    a, b, c = U[:-2, 1:-1, 1:-1], U[2:, 1:-1, 1:-1], U[1:-1, 1:-1, 1:-1]
    V[1:-1, 1:-1, 1:-1] = (a + b) * (a + b) - c
    return [V]


def regs_want(x):
    u = x["u"]
    v = onp.zeros(u.shape, u.dtype)
    s = u[:-2, 1:-1, 1:-1] + u[2:, 1:-1, 1:-1]
    v[1:-1, 1:-1, 1:-1] = s * s - u[1:-1, 1:-1, 1:-1]
    return [v]


case("registers_f32", {"u": edge_data((20, 30, 132), F32, 70)}, regs_run, regs_want,
     ["MOV.F32", "MOV.F32", "ADD.F32", "ADD.F32", "MULRSUB.F32"], {"kernel": "stencil_tile", "elem": "4", "loader": "cp.async"})


def abs_run(np, X):
    U = X["u"]
    V = np.zeros(U.shape, dtype=U.dtype)
    V[1:-1, 1:-1, 1:-1] = abs(U[:-2, 1:-1, 1:-1] - U[2:, 1:-1, 1:-1]) * U[1:-1, 1:-1, 1:-1]
    return [V]


def abs_want(x):
    u = x["u"]
    v = onp.zeros(u.shape, u.dtype)
    v[1:-1, 1:-1, 1:-1] = onp.abs(u[:-2, 1:-1, 1:-1] - u[2:, 1:-1, 1:-1]) * u[1:-1, 1:-1, 1:-1]
    return [v]


for dt in (F32, F64):
    case("abs_%s" % dt.__name__, {"u": edge_data((20, 30, 131), dt, 71)}, abs_run, abs_want,
         ["SUB.%s" % _cls(dt), "ABS.%s" % _cls(dt), "MUL.%s" % _cls(dt)], {"kernel": "stencil_tile", "elem": "4" if dt == F32 else "8"})


# ---- sstencil / @stencil ----------------------------------------------------------------------------------------------------
def _st_star(a):
    return 0.25 * (a[-1, 0] + a[1, 0] + a[0, -1] + a[0, 1]) + a[0, 0]


def _st_asym(a):
    return a[-2, 0] + a[0, 3] - 0.5 * a[1, -1]


def _st_limit(a):
    return a[0, -8] + a[0, 8] + a[8, 0] + a[-8, 0]


def _st_beyond(a):
    return a[0, -8] + a[0, 9] + a[1, 0]


def st_star_want(x):
    v = onp.zeros(x.shape, F64)
    v[1:-1, 1:-1] = 0.25 * (((x[:-2, 1:-1] + x[2:, 1:-1]) + x[1:-1, :-2]) + x[1:-1, 2:]) + x[1:-1, 1:-1]
    return v


def st_asym_want(x):
    n, m = x.shape
    v = onp.zeros(x.shape, F64)
    v[2:n - 1, 1:m - 3] = (x[0:n - 3, 1:m - 3] + x[2:n - 1, 4:m]) - 0.5 * x[3:n, 0:m - 4]
    return v


def st_limit_want(x):
    n, m = x.shape
    v = onp.zeros(x.shape, F64)
    v[8:n - 8, 8:m - 8] = ((x[8:n - 8, 0:m - 16] + x[8:n - 8, 16:m]) + x[16:n, 8:m - 8]) + x[0:n - 16, 8:m - 8]
    return v


def st_beyond_want(x):
    n, m = x.shape
    v = onp.zeros(x.shape, F64)
    v[0:n - 1, 8:m - 9] = (x[0:n - 1, 0:m - 17] + x[0:n - 1, 17:m]) + x[1:n, 8:m - 9]
    return v


def sst_run(np, X, f):
    return [np.sstencil(np.stencil(f), X["x"])]


for nm, f, w, ops, plan in [
        ("star", _st_star, st_star_want, ["ADD.F64"] * 3 + ["MULADD.F64"], {"kernel": "stencil_terms", "staged_views": "5"}),
        ("asym", _st_asym, st_asym_want, ["ADD.F64", "MULSUB.F64"], {"kernel": "stencil_terms", "halo": "z0+0,y0+3,x1+3"}),
        ("limit", _st_limit, st_limit_want, ["ADD.F64"] * 3, {"kernel": "stencil_terms", "halo": "z0+0,y8+8,x0+8", "staged_views": "3"}),
        ("beyond", _st_beyond, st_beyond_want, ["ADD.F64"] * 2, {"kernel": "stencil_terms", "staged_views": "2"})]:
    case("sstencil_%s" % nm, {"x": edge_data((150, 290), F64, 80)}, lambda np, X, f=f: sst_run(np, X, f),
         lambda x, w=w: [w(x["x"])], ops, plan)


def sst_chain_run(np, X):
    x = X["x"]
    s1 = np.sstencil(np.stencil(_st_star), x)  # allocated like x: padded shards, zero border
    out = np.full(x.shape, 7.0, local_border=2)
    np.sstencil(np.stencil(_st_asym), s1, out=out)  # out= keeps its border
    return [s1, out]


def sst_chain_want(x):
    s1 = st_star_want(x["x"])
    out = onp.full(s1.shape, 7.0)
    inner = st_asym_want(s1)
    n, m = s1.shape
    out[2:n - 1, 1:m - 3] = inner[2:n - 1, 1:m - 3]
    return [s1, out]


case("sstencil_chain_local_border", {"x": edge_data((130, 150), F64, 81)}, sst_chain_run, sst_chain_want,
     ["ADD.F64", "MULSUB.F64"], {"kernel": "stencil_terms"}, border={"local_border": 2})


# ---- running a case -----------------------------------------------------------------------------------------------------
def _fields(plan):
    return dict(kv.split("=", 1) for kv in plan.split() if "=" in kv)


def evaluate(c):
    """(outputs as host arrays, [[plan, ['OP.CLASS', ...], n_regs], ...] of every op list the run handed to the backend)"""
    import ramba_b200 as rb
    from ramba_b200 import _cabi
    from ramba_b200.runtime import RT

    X = {k: rb.fromarray(v, **(c.border or {})) for k, v in c.inputs.items()}
    rb.sync()
    be = RT.be()
    run, seen = be.run, []
    cls = {0: "F64", 1: "F32", 2: "I64"}

    def record(fop, stream=None):
        ops = ["%s.%s" % (_cabi.OPS[fop.insns[i].op], cls[fop.insns[i].ctype]) for i in range(fop.n_insns)]
        seen.append([_cabi.describe_plan(fop), ops, int(fop.n_regs)])
        return run(fop, stream)

    be.run = record
    try:
        outs = c.run(rb, X)
        rb.sync()
        got = [o.asarray() for o in outs]
    finally:
        be.run = run
    return got, seen


def case_failures(c, got, seen, plan_fields=True):
    with onp.errstate(all="ignore"):
        fails = mismatches(got, c.want(c.inputs), c.name)
    mine = [p for p, ops, _ in seen if ops == c.ops]
    if not mine:
        fails.append("%s: no op list is %s: %s" % (c.name, c.ops, [s[1] for s in seen]))
    elif plan_fields:
        f = _fields(mine[-1])
        f["kernel"] = mine[-1].split()[0][len("kernel="):]
        bad = {k: (f.get(k), v) for k, v in c.plan.items() if f.get(k) != v}
        if bad:
            fails.append("%s: plan %s: (got, want) %s" % (c.name, mine[-1], bad))
    return fails, mine


def _derived(plan):
    """the facts each plan line implies: prefetch = ring - z halo - 1"""
    f = _fields(plan)
    if plan.startswith("kernel=stencil_") and f["loader"] != "none":
        z = f["halo"].split(",")[0][1:].split("+")
        return {"prefetch": int(f["ring"]) - int(z[0]) - int(z[1]) - 1}
    return {}


# what each switch set must keep every op list off, and what it must still reach
SWITCHES = {"default": {}, "no_terms": {"RB200_NO_TERMS_KERNEL": "1"}, "no_tma": {"RB200_NO_TMA": "1"},
            "no_tile": {"RB200_NO_TILE_KERNEL": "1"}}
BARRED = {"no_terms": lambda p: p.startswith("kernel=stencil_terms"), "no_tma": lambda p: " loader=tma " in p,
          "no_tile": lambda p: p.startswith("kernel=stencil_")}
REACHED = {"no_terms": lambda p: p.startswith("kernel=stencil_tile ") and " loader=tma " in p,
           "no_tma": lambda p: p.startswith("kernel=stencil_terms ") and " loader=cp.async " in p,
           "no_tile": lambda p: p.startswith("kernel=general_interpreter")}


def run_cases(switches, names=None):
    """{case: [failures, [plans of its op lists]]} of every case in this process"""
    out = {}
    for c in CASES:
        if names and c.name not in names:
            continue
        print("case", c.name, flush=True)  # (the last name printed is the case a failing process was running)
        got, seen = evaluate(c)
        fails, _ = case_failures(c, got, seen, plan_fields=switches == "default")
        out[c.name] = [fails, [s[0] for s in seen]]
        del got
    return out


def check_run(switches, out):
    fails = [f for v in out.values() for f in v[0]]
    plans = [p for v in out.values() for p in v[1]]
    if switches == "default":
        # together the cases reach every plan form of the two kernels
        need = {"kernel=stencil_terms ": 1, "kernel=stencil_tile ": 1, " loader=tma ": 1, " loader=cp.async ": 1,
                " loader=none ": 1, " elem=4 ": 1, " elem=8 ": 1, "(f32:0) ": 1, " fast_tail=1 ": 1, " chains=1 ": 1}
        for k in need:
            if not any(k in p for p in plans if p.startswith("kernel=stencil_")):
                fails.append("no plan has %r" % k)
        terms = [_fields(p) for p in plans if p.startswith("kernel=stencil_terms ")]
        if not any(f["terms"].split("(")[0] == f["terms"].split(":")[1][:-1] for f in terms):
            fails.append("no plan runs every term in float32")
        if not any(f["fast_tail"] == "0" and 0 < int(f["terms"].split(":")[1][:-1]) < int(f["terms"].split("(")[0]) for f in terms):
            fails.append("no split plan without the fast tail")
        pf = {_derived(p).get("prefetch") for p in plans}
        if not {1, 2} <= pf:
            fails.append("prefetch 1 and 2 not both reached: %s" % pf)
        # no plan hands the term kernel a float32 phase over float64 staged data
        for p in plans:
            f = _fields(p)
            if p.startswith("kernel=stencil_terms ") and f["elem"] == "8" and not f["terms"].endswith("(f32:0)"):
                fails.append("term kernel with elem=8 and a float32 phase: %s" % p)
    else:
        fails += ["%s: %s" % (switches, p) for p in plans if BARRED[switches](p)]
        if not any(REACHED[switches](p) for p in plans):
            fails.append("%s: the fall-back form was never reached" % switches)
    return fails


@pytest.mark.parametrize("c", CASES, ids=lambda c: c.name)
def test_oracle_against_reference(oracle_engine, c):
    """the op list the engine builds means what the case's NumPy expression says, bit for bit, on the plan it names"""
    got, seen = evaluate(c)
    fails, mine = case_failures(c, got, seen)
    assert not fails, fails
    for p in mine:
        if p.startswith("kernel=stencil_") and " items=" in p and c.name.startswith("zhalo"):
            f = _fields(p)
            assert int(f["items"]) > int(f["ctas"]) and int(f["planes_per_item"]) < int(f["box"].split("x")[0]), p


def test_plan_coverage_on_the_oracle(oracle_engine):
    out = {}
    for c in CASES:
        _, seen = evaluate(c)
        out[c.name] = [[], [s[0] for s in seen]]
    fails = check_run("default", out)
    assert not fails, fails


def test_float32_prefix_never_reaches_the_float64_term_kernel(oracle_engine):
    """the planner refused the term form for a float64 group behind a float32 prefix: stencil_terms_kernel<double> has
    no float32 phase and stored nothing"""
    c = next(c for c in CASES if c.name == "f32_prefix_f64_group")
    got, seen = evaluate(c)
    assert not case_failures(c, got, seen)[0]
    assert not any(p.startswith("kernel=stencil_terms") for p, _, _ in seen), seen


# ---- kernel switches, one process each ------------------------------------------------------------------------------------
def _switched_worker(out_path, switches, backend):
    from ramba_b200.runtime import RT

    RT.reset()
    if backend == "oracle":
        import _oracle_backend

        _oracle_backend.install()
    elif os.environ.get("RB200_DRY_GPU_TESTS"):
        import conftest

        conftest._dry_gpu()
    out = run_cases(switches)
    if backend == "gpu":
        from ramba_b200 import _cabi

        assert RT.is_cuda and _cabi.launch_count() > 0, "the CUDA library did not run"
    with open(out_path, "w") as f:
        json.dump(out, f)


def _run_switched(tmp_path, switches, backend):
    path = str(tmp_path / ("%s_%s.json" % (switches, backend)))
    code = "import sys; sys.path[:0] = [%r, %r]; import test_stencil_semantics as t; t._switched_worker(%r, %r, %r)" % (
        ROOT, HERE, path, switches, backend)
    env = dict(os.environ, **SWITCHES[switches])
    r = subprocess.run([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-3000:]
    with open(path) as f:
        return json.load(f)


@pytest.mark.parametrize("switches", [s for s in SWITCHES if s != "default"])
def test_switched_kernels_on_the_oracle(tmp_path, switches):
    out = _run_switched(tmp_path, switches, "oracle")
    fails = check_run(switches, out)
    assert not fails, fails[:10]


@pytest.mark.gpu
@pytest.mark.timeout(3000)
@pytest.mark.parametrize("switches", list(SWITCHES))
def test_cases_on_the_gpu(tmp_path, switches):
    out = _run_switched(tmp_path, switches, "gpu")
    fails = check_run(switches, out)
    assert not fails, fails[:10]


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_float32_laplacian_past_2_31_elements(gpu_engine):
    """7-point float32 Laplacian over 2050 x 1026 x 1026 (2.16e9 elements, 8.6 GB each for U and V).  U is generated on
    the device from the indices; the first, last and the planes around linear index 2^31 are checked against the
    reference."""
    import ramba_b200 as rb
    from ramba_b200 import _cabi

    Z, Y, X = 2050, 1026, 1026
    assert Z * Y * X > 2 ** 31

    def gen(i, j, k):
        return ((i * 7 + j * 13 + k * 5) % 31 - 15) * 0.1

    U = rb.fromfunction(gen, (Z, Y, X), dtype=F32)
    V = rb.zeros((Z, Y, X), dtype=F32)
    rb.sync()
    before = _cabi.launch_count()
    V[1:-1, 1:-1, 1:-1] = (U[:-2, 1:-1, 1:-1] + U[2:, 1:-1, 1:-1] + U[1:-1, :-2, 1:-1] + U[1:-1, 2:, 1:-1]
                           + U[1:-1, 1:-1, :-2] + U[1:-1, 1:-1, 2:] - 6.0 * U[1:-1, 1:-1, 1:-1])
    rb.sync()
    assert _cabi.launch_count() > before
    zc = 2 ** 31 // (Y * X)
    fails = []
    for z in sorted({0, 1, zc - 1, zc, zc + 1, Z - 2, Z - 1}):
        lo, hi = max(z - 1, 0), min(z + 2, Z)
        i, j, k = onp.meshgrid(onp.arange(lo, hi), onp.arange(Y), onp.arange(X), indexing="ij")
        u = gen(i, j, k).astype(F32)  # the same float64 formula, stored to float32
        assert onp.array_equal(u, U[lo:hi].asarray()), z
        want = onp.zeros((Y, X), F32)
        if 0 < z < Z - 1:
            want = lap_want(u, F32)[0][z - lo] if hi - lo == 3 else want
        fails += mismatches([V[z].asarray()], [want], "plane %d" % z)
    assert not fails, fails


# ---- each check rejects a wrong restatement fed through the same comparison ------------------------------------------
def _wrong_f64_phase(x):
    u = c64(x["u"])  # the float32 neighbour sum done in float64
    return lap_want(u, F32, out=onp.zeros(u.shape, F32))


def _wrong_dropped_term(x):
    u = x["u"]
    v = onp.zeros(u.shape, F32)
    s = (((u[:-2, 1:-1, 1:-1] + u[2:, 1:-1, 1:-1]) + u[1:-1, :-2, 1:-1]) + u[1:-1, 2:, 1:-1]) + u[1:-1, 1:-1, :-2]
    v[1:-1, 1:-1, 1:-1] = (c64(s) - 6.0 * c64(u[1:-1, 1:-1, 1:-1])).astype(F32)
    return [v]


def _wrong_halo(x):
    u = x["u"]
    v = onp.zeros(u.shape, F32)
    s = ((((u[:-2, 1:-1, 1:-1] + u[2:, 1:-1, 1:-1]) + u[1:-1, :-2, 1:-1]) + u[1:-1, 2:, 1:-1]) + u[1:-1, 1:-1, 1:-1]) + u[1:-1, 1:-1, 2:]
    v[1:-1, 1:-1, 1:-1] = (c64(s) - 6.0 * c64(u[1:-1, 1:-1, 1:-1])).astype(F32)
    return [v]


def _wrong_fma(x):
    u = x["u"]
    v = onp.zeros(u.shape, F64)
    v[1:-1, 1:-1] = fma64(-0.1, u[1:-1, 1:-1], 0.3 * u[:-2, 1:-1] + 0.7 * u[2:, 1:-1])
    return [v]


def _wrong_border(x):
    s1, out = sst_chain_want(x)
    n, m = out.shape
    keep = out[2:n - 1, 1:m - 3].copy()
    out[:] = 0.0  # the border written as sstencil's own zeros
    out[2:n - 1, 1:m - 3] = keep
    return [s1, out]


WRONG = [("lap_tma_f32", "float32 phase in float64", _wrong_f64_phase), ("lap_tma_f32", "dropped term", _wrong_dropped_term),
         ("lap_tma_f32", "halo off by one", _wrong_halo), ("weighted_float64", "contracted multiply-add", _wrong_fma),
         ("sstencil_chain_local_border", "border overwritten", _wrong_border)]


@pytest.mark.parametrize("name,what,wrong", WRONG, ids=[w[1].replace(" ", "_") for w in WRONG])
def test_checks_reject_wrong_restatements(oracle_engine, name, what, wrong):
    c = next(c for c in CASES if c.name == name)
    got, seen = evaluate(c)
    assert not case_failures(c, got, seen)[0]
    with onp.errstate(all="ignore"):
        assert mismatches(got, wrong(c.inputs), name), "%s: the check does not see a %s" % (name, what)


# ---- several ranks ---------------------------------------------------------------------------------------------------------
# every axis is cut in some world: the partitioner splits the longest dimensions first
case("world_lap_z_f32", {"u": edge_data((64, 18, 20), F32, 90)}, lap_run, lambda x: lap_want(x["u"], F32), LAP_OPS[F32])
case("world_lap_y_f64", {"u": edge_data((10, 66, 24), F64, 91)}, lap_run, lambda x: lap_want(x["u"], F64), LAP_OPS[F64])
case("world_lap_x_f32", {"u": edge_data((8, 14, 300), F32, 92)}, lap_run, lambda x: lap_want(x["u"], F32), LAP_OPS[F32])
case("world_sum4_rows_f32", {"u": edge_data((300, 40), F32, 93)}, sum4_2d_run, lambda x: sum4_2d_want(x["u"]), ["ADD.F32"] * 3)
WORLD_CASES = ["world_lap_z_f32", "world_lap_y_f64", "world_lap_x_f32", "world_sum4_rows_f32", "f32_prefix_f64_group",
               "f32_overflow_before_promotion", "split_no_fast_tail_f32", "halo_xspan16_f32", "sstencil_asym",
               "sstencil_chain_local_border", "direct_kinds_f32", "lap_local_border_f64"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run_world(world, out):
    port = _free_port()
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), OMP_NUM_THREADS="1")
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_stencil_worker.py"), out], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=900)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, o))
    for rc, o in outs:
        assert rc == 0, o[-3000:]
    return dict(onp.load(out))


@pytest.fixture(scope="module")
def stencil_worlds(tmp_path_factory):
    d = tmp_path_factory.mktemp("stencil_worlds")
    return {w: _run_world(w, str(d / ("w%d.npz" % w))) for w in (1, 2, 3, 4, 8)}


@pytest.mark.timeout(1800)
def test_worlds_match_one_rank_and_the_reference(stencil_worlds):
    fails, cut = [], set()
    for w, res in stencil_worlds.items():
        for name in WORLD_CASES:
            c = next(c for c in CASES if c.name == name)
            with onp.errstate(all="ignore"):
                want = c.want(c.inputs)
            got = [res["%s.%d" % (name, i)] for i in range(len(want))]
            fails += mismatches(got, want, "W=%d %s" % (w, name))
            fails += mismatches(got, [stencil_worlds[1]["%s.%d" % (name, i)] for i in range(len(want))], "W=%d %s against W=1" % (w, name))
            blocks = res[name + ".blocks"]
            nd = blocks.shape[1] // 2
            for d in range(nd):
                if len({int(b[d]) for b in blocks if (b[nd:] > 0).all()}) > 1:
                    cut.add((w, nd, d))
    assert not fails, fails[:10]
    # halos cross rank boundaries along every axis of the 3-D cases, and along the rows of the 2-D ones, in every world
    for w in (2, 3, 4, 8):
        assert {(3, 0), (3, 1), (3, 2), (2, 0)} <= {(nd, d) for ww, nd, d in cut if ww == w}, (w, sorted(cut))
