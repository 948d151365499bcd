"""ctypes binding of libramba_b200.so (include/ramba_b200.h).

This is the thin C-ABI the deferred-op fuser dispatches through.  The reference ships Python
source to its workers and lets Numba compile it (ramba/ramba.py:3526-3545, 249-438); here the
worker side is a prebuilt sm_90a library and the "kernel source" is an op list.

There is no fallback: if the library is missing or no CUDA device is usable, loading or launching
raises.
"""
import ctypes as C
import os

ABI_VERSION = 7
MAX_DIMS = 5
MAX_VIEWS = 16
MAX_SCALARS = 32
MAX_INSNS = 96
MAX_REGS = 12
MAX_REDS = 4
NOSTORE = 0xFF

# storage dtypes
F64, F32, I64, I32, BOOL, U8, I8, I16, U16, U32 = range(10)
# compute classes
T_F64, T_F32, T_I64 = range(3)
# operand kinds
K_NONE, K_ACC, K_REG, K_VIEW, K_SCAL, K_IOTA = range(6)

OPS = [
    "MOV", "ADD", "SUB", "MUL", "DIV", "FLOORDIV", "MOD", "POW", "POWI", "MIN", "MAX",
    "GT", "LT", "GE", "LE", "EQ", "NE", "LAND", "LOR", "LXOR", "BAND", "BOR", "BXOR", "SHL", "SHR",
    "ABS", "SQUARE", "SQRT", "SIN", "COS", "TAN", "SINH", "COSH", "TANH", "ASIN", "ACOS", "ATAN",
    "NEG", "EXP", "LOG", "ISFINITE", "ISINF", "ISNAN", "ISNEGINF", "ISPOSINF", "LNOT", "INVERT",
    "WHERE", "CVT", "SINCOS", "RED", "CBRT", "MULADD", "MULSUB", "MULRSUB", "PHILOX",
]
OP = {name: i for i, name in enumerate(OPS)}
RED_ADD, RED_MUL, RED_MIN, RED_MAX = range(4)
# output forms of PHILOX (imm)
PHILOX_UNIFORM64, PHILOX_UNIFORM32, PHILOX_NORMAL64, PHILOX_INTEGER = range(4)
# grouped-reduction ops (rb200_group_reduce)
GROUP_SUM, GROUP_PROD, GROUP_MIN, GROUP_MAX, GROUP_NANSUM, GROUP_NANCOUNT, GROUP_SQDEV = range(7)
# index-reduction ops (rb200_arg_reduce) and its "every axis" value of `axis`
ARG_MAX, ARG_MIN, ARG_NANMAX, ARG_NANMIN = range(4)
ARG_ALL_AXES = -1
# stream-compaction payload forms (rb200_compact) and its chunk size
COMPACT_VALUES, COMPACT_FLAT, COMPACT_COORDS = range(3)
COMPACT_CHUNK = 4096
# binning: bin-table forms (rb200_histogram) and search sides (rb200_bin_search)
BINS_UNIFORM, BINS_EDGES, BINS_INTEGER = range(3)
SEARCH_LEFT, SEARCH_RIGHT = range(2)
# order statistics: count-pass modes (rb200_select_count)
SELECT_READ, SELECT_APPEND, SELECT_CAND = range(3)


class Insn(C.Structure):
    _fields_ = [
        ("op", C.c_uint8), ("ctype", C.c_uint8),
        ("a_kind", C.c_uint8), ("a_idx", C.c_uint8),
        ("b_kind", C.c_uint8), ("b_idx", C.c_uint8),
        ("c_kind", C.c_uint8), ("c_idx", C.c_uint8),
        ("st_reg", C.c_uint8), ("st_view", C.c_uint8),
        ("st2", C.c_uint8), ("mask_reg", C.c_uint8),
        ("imm", C.c_uint32),
    ]


class View(C.Structure):
    _fields_ = [
        ("base", C.c_void_p),
        ("stride", C.c_int64 * MAX_DIMS),
        ("dtype", C.c_int32),
        ("flags", C.c_int32),
        ("alloc_lo", C.c_void_p),
        ("alloc_hi", C.c_void_p),
    ]


class Red(C.Structure):
    _fields_ = [
        ("op", C.c_int32), ("ctype", C.c_int32),
        ("out", C.c_void_p),
        ("out_dtype", C.c_int32), ("pad", C.c_int32),
    ]


class FusedOp(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("ndim", C.c_int32),
        ("itershape", C.c_int64 * MAX_DIMS),
        ("global_start", C.c_int64 * MAX_DIMS),
        ("iota_dim", C.c_int32 * MAX_DIMS),
        ("worker_num", C.c_int32), ("num_workers", C.c_int32),
        ("n_views", C.c_int32), ("n_scalars", C.c_int32), ("n_insns", C.c_int32),
        ("n_regs", C.c_int32), ("n_reds", C.c_int32),
        ("n_axis_red_dims", C.c_int32), ("axis_nsplit", C.c_int32),
        ("views", View * MAX_VIEWS),
        ("scalars", C.c_uint64 * MAX_SCALARS),
        ("insns", Insn * MAX_INSNS),
        ("reds", Red * MAX_REDS),
        ("red_scratch", C.c_void_p),
    ]


class IndexView(C.Structure):
    _fields_ = [
        ("base", C.c_void_p),
        ("ndim", C.c_int32), ("elem_bytes", C.c_int32),
        ("shape", C.c_int64 * MAX_DIMS),
        ("stride", C.c_int64 * MAX_DIMS),
        ("alloc_lo", C.c_void_p),
        ("alloc_hi", C.c_void_p),
    ]


class BinTable(C.Structure):
    _fields_ = [
        ("form", C.c_int32), ("edge_dtype", C.c_int32),
        ("n_bins", C.c_int64),
        ("edges", C.c_void_p),
        ("lo_dtype", C.c_int32), ("hi_dtype", C.c_int32), ("sub_dtype", C.c_int32), ("div_dtype", C.c_int32),
        ("lo", C.c_double), ("hi", C.c_double),
        ("lo_i", C.c_int64), ("hi_i", C.c_int64),
        ("first", C.c_double), ("denom", C.c_double),
    ]


class SelectState(C.Structure):
    _fields_ = [
        ("segments", C.c_int64), ("targets", C.c_int64),
        ("rank", C.c_void_p), ("key", C.c_void_p), ("slot", C.c_void_p), ("slot_key", C.c_void_p), ("n_slots", C.c_void_p),
        ("counts", C.c_void_p), ("nans", C.c_void_p), ("matched", C.c_void_p), ("cand", C.c_void_p),
        ("cand_cap", C.c_int64),
        ("cand_n", C.c_void_p),
        ("seg_dims", C.c_int32),
        ("seg_shape", C.c_int64 * MAX_DIMS), ("seg_gstride", C.c_int64 * MAX_DIMS),
        ("seg_base", C.c_int64),
    ]


class RouteTable(C.Structure):
    _fields_ = [
        ("ndim", C.c_int32), ("n_ranks", C.c_int32),
        ("shape", C.c_int64 * MAX_DIMS),
        ("n_cells", C.c_int32 * MAX_DIMS),
        ("cut_start", C.c_int32 * MAX_DIMS),
        ("cuts", C.c_void_p),
        ("cell_owner", C.c_void_p),
        ("cell_offset", C.c_void_p),
        ("cell_stride", C.c_void_p),
    ]


class GroupTable(C.Structure):
    _fields_ = [
        ("n_groups", C.c_int32),
        ("len", C.c_int64),
        ("offsets", C.c_void_p),
        ("members", C.c_void_p),
    ]


assert C.sizeof(Insn) == 16

# every symbol include/ramba_b200.h declares
EXPORTS = [
    "rb200_run_deferred_ops",
    "rb200_red_scratch_bytes",
    "rb200_reduce_partials",
    "rb200_cumulative",
    "rb200_cumulative_scratch_bytes",
    "rb200_describe_plan",
    "rb200_last_error",
    "rb200_abi_version",
    "rb200_launch_count",
    "rb200_reset_launch_count",
    "rb200_device_sm_count",
    "rb200_gather",
    "rb200_scatter",
    "rb200_route",
    "rb200_route_scratch_bytes",
    "rb200_group_reduce",
    "rb200_group_reduce_scratch_bytes",
    "rb200_describe_group_plan",
    "rb200_arg_reduce",
    "rb200_arg_reduce_scratch_bytes",
    "rb200_describe_arg_plan",
    "rb200_compact_count",
    "rb200_compact",
    "rb200_describe_compact_plan",
    "rb200_histogram",
    "rb200_histogram_scratch_bytes",
    "rb200_describe_hist_plan",
    "rb200_bin_search",
    "rb200_select_count",
    "rb200_select_choose",
    "rb200_select_rows",
    "rb200_select_scratch_bytes",
    "rb200_describe_select_plan",
]

_LIB = None


def lib_path():
    # RAMBA_B200_LIB: A/B-test another build of the same ABI (development aid)
    return os.environ.get("RAMBA_B200_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libramba_b200.so")


class CabiError(RuntimeError):
    pass


def load():
    """Load libramba_b200.so; raises (loudly) if it was not built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        raise CabiError(
            "libramba_b200.so not found at %s — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback)" % path
        )
    lib = C.CDLL(path)
    lib.rb200_run_deferred_ops.argtypes = [C.POINTER(FusedOp), C.c_void_p]
    lib.rb200_run_deferred_ops.restype = C.c_int
    lib.rb200_red_scratch_bytes.argtypes = []
    lib.rb200_red_scratch_bytes.restype = C.c_int64
    lib.rb200_reduce_partials.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_void_p]
    lib.rb200_reduce_partials.restype = C.c_int
    lib.rb200_cumulative.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p]
    lib.rb200_cumulative.restype = C.c_int
    lib.rb200_cumulative_scratch_bytes.argtypes = [C.c_int64, C.c_int64, C.c_int64]
    lib.rb200_cumulative_scratch_bytes.restype = C.c_int64
    lib.rb200_describe_plan.argtypes = [C.POINTER(FusedOp), C.c_char_p, C.c_int64]
    lib.rb200_describe_plan.restype = C.c_int
    lib.rb200_last_error.argtypes = []
    lib.rb200_last_error.restype = C.c_char_p
    lib.rb200_abi_version.argtypes = []
    lib.rb200_abi_version.restype = C.c_int
    lib.rb200_launch_count.argtypes = []
    lib.rb200_launch_count.restype = C.c_int64
    lib.rb200_reset_launch_count.argtypes = []
    lib.rb200_reset_launch_count.restype = None
    lib.rb200_device_sm_count.argtypes = []
    lib.rb200_device_sm_count.restype = C.c_int
    lib.rb200_gather.argtypes = [C.POINTER(IndexView), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.rb200_gather.restype = C.c_int
    lib.rb200_scatter.argtypes = [C.POINTER(IndexView), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.rb200_scatter.restype = C.c_int
    lib.rb200_route.argtypes = [C.POINTER(RouteTable), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p]
    lib.rb200_route.restype = C.c_int
    lib.rb200_route_scratch_bytes.argtypes = [C.c_int64, C.c_int32]
    lib.rb200_route_scratch_bytes.restype = C.c_int64
    lib.rb200_group_reduce.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int32, C.POINTER(GroupTable), C.c_int32, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p]
    lib.rb200_group_reduce.restype = C.c_int
    lib.rb200_group_reduce_scratch_bytes.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int32]
    lib.rb200_group_reduce_scratch_bytes.restype = C.c_int64
    lib.rb200_describe_group_plan.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int32]
    lib.rb200_describe_group_plan.restype = C.c_char_p
    lib.rb200_arg_reduce.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p]
    lib.rb200_arg_reduce.restype = C.c_int
    lib.rb200_arg_reduce_scratch_bytes.argtypes = [C.POINTER(IndexView), C.c_int32]
    lib.rb200_arg_reduce_scratch_bytes.restype = C.c_int64
    lib.rb200_describe_arg_plan.argtypes = [C.POINTER(IndexView), C.c_int32]
    lib.rb200_describe_arg_plan.restype = C.c_char_p
    lib.rb200_compact_count.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]
    lib.rb200_compact_count.restype = C.c_int
    lib.rb200_compact.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.rb200_compact.restype = C.c_int
    lib.rb200_describe_compact_plan.argtypes = [C.POINTER(IndexView), C.c_int64]
    lib.rb200_describe_compact_plan.restype = C.c_char_p
    lib.rb200_histogram.argtypes = [C.POINTER(IndexView), C.c_int32, C.POINTER(IndexView), C.c_int32, C.POINTER(BinTable), C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p]
    lib.rb200_histogram.restype = C.c_int
    lib.rb200_histogram_scratch_bytes.argtypes = [C.POINTER(IndexView), C.c_int32, C.POINTER(BinTable)]
    lib.rb200_histogram_scratch_bytes.restype = C.c_int64
    lib.rb200_describe_hist_plan.argtypes = [C.POINTER(IndexView), C.c_int32, C.POINTER(BinTable)]
    lib.rb200_describe_hist_plan.restype = C.c_char_p
    lib.rb200_bin_search.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.rb200_bin_search.restype = C.c_int
    lib.rb200_select_count.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int64, C.POINTER(SelectState), C.c_int32, C.c_int32, C.c_void_p]
    lib.rb200_select_count.restype = C.c_int
    lib.rb200_select_choose.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int64, C.POINTER(SelectState), C.c_int32, C.c_void_p]
    lib.rb200_select_choose.restype = C.c_int
    lib.rb200_select_rows.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int64, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                      C.c_void_p]
    lib.rb200_select_rows.restype = C.c_int
    lib.rb200_select_scratch_bytes.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int64, C.c_int64, C.c_int64]
    lib.rb200_select_scratch_bytes.restype = C.c_int64
    lib.rb200_describe_select_plan.argtypes = [C.POINTER(IndexView), C.c_int32, C.c_int64, C.c_int64, C.c_int64]
    lib.rb200_describe_select_plan.restype = C.c_char_p
    if lib.rb200_abi_version() != ABI_VERSION:
        raise CabiError("libramba_b200.so ABI %d != binding ABI %d: rebuild" % (lib.rb200_abi_version(), ABI_VERSION))
    _LIB = lib
    return lib


def check(rc):
    if rc != 0:
        raise CabiError("libramba_b200: " + load().rb200_last_error().decode("utf-8", "replace"))


def run_deferred_ops(fop, stream=None):
    """Launch one fused op over one range (FusedOp struct) on a cudaStream_t handle (int or None)."""
    lib = load()
    check(lib.rb200_run_deferred_ops(C.byref(fop), C.c_void_p(stream) if stream else None))


def reduce_partials(out_ptr, part_ptr, n, k, stride_k, dtype, redop, stream=None):
    lib = load()
    check(lib.rb200_reduce_partials(C.c_void_p(out_ptr), C.c_void_p(part_ptr), n, k, stride_k, dtype, redop,
                                    C.c_void_p(stream) if stream else None))


def cumulative(src, dst, dtype, n_outer, length, n_inner, redop, carry_in=None, totals_out=None, scratch=None, stream=None):
    """Inclusive scan of one block [n_outer][length][n_inner] along `length` (device pointers as ints)."""
    lib = load()
    check(lib.rb200_cumulative(C.c_void_p(src), C.c_void_p(dst), dtype, n_outer, length, n_inner, redop,
                               C.c_void_p(carry_in) if carry_in else None, C.c_void_p(totals_out) if totals_out else None,
                               C.c_void_p(scratch) if scratch else None, C.c_void_p(stream) if stream else None))


def cumulative_scratch_bytes(n_outer, length, n_inner):
    return int(load().rb200_cumulative_scratch_bytes(n_outer, length, n_inner))


def describe_plan(fop):
    """One text line: the kernel the library would run this fused op on, and how (no device needed)."""
    lib = load()
    buf = C.create_string_buffer(600)
    check(lib.rb200_describe_plan(C.byref(fop), buf, 600))
    return buf.value.decode()


def red_scratch_bytes():
    return int(load().rb200_red_scratch_bytes())


def launch_count():
    return int(load().rb200_launch_count())


def reset_launch_count():
    load().rb200_reset_launch_count()


def index_view(base, shape, strides, elem_bytes, bounds=None):
    """An IndexView struct: element (c0..) at base + elem_bytes * sum(c_d * strides[d]) (device addresses as ints)."""
    v = IndexView()
    v.base = base
    v.ndim = len(shape)
    v.elem_bytes = elem_bytes
    for d, (n, s) in enumerate(zip(shape, strides)):
        v.shape[d] = int(n)
        v.stride[d] = int(s)
    if bounds is not None:
        v.alloc_lo, v.alloc_hi = bounds
    return v


def route_table(shape, cuts, owners, offsets, strides, n_ranks):
    """A RouteTable struct over host arrays: cuts is a list (per dim) of ascending cut points, owners / offsets one entry
    per cell (C order over the cell grid), strides ndim entries per cell.  Returns (struct, arrays to keep alive)."""
    import numpy as np

    k = len(shape)
    flat_cuts = np.ascontiguousarray(np.concatenate([np.asarray(c, dtype=np.int64) for c in cuts]), dtype=np.int64)
    own = np.ascontiguousarray(owners, dtype=np.int32)
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    st = np.ascontiguousarray(np.asarray(strides, dtype=np.int64).reshape(-1))
    t = RouteTable()
    t.ndim = k
    t.n_ranks = n_ranks
    start = 0
    for d in range(k):
        t.shape[d] = int(shape[d])
        t.n_cells[d] = len(cuts[d]) - 1
        t.cut_start[d] = start
        start += len(cuts[d])
    t.cuts, t.cell_owner, t.cell_offset, t.cell_stride = flat_cuts.ctypes.data, own.ctypes.data, off.ctypes.data, st.ctypes.data
    return t, (flat_cuts, own, off, st)


def _p(x):
    return C.c_void_p(x) if x else None


def gather(view, lin, n, out, bad, stream=None):
    check(load().rb200_gather(C.byref(view), _p(lin), n, _p(out), _p(bad), _p(stream)))


def scatter(view, lin, n, values, bad, stream=None):
    check(load().rb200_scatter(C.byref(view), _p(lin), n, _p(values), _p(bad), _p(stream)))


def route(table, lin, n, offsets, slots, counts, bad, scratch, stream=None):
    check(load().rb200_route(C.byref(table), _p(lin), n, _p(offsets), _p(slots), _p(counts), _p(bad), _p(scratch), _p(stream)))


def route_scratch_bytes(n, n_ranks):
    return int(load().rb200_route_scratch_bytes(n, n_ranks))


def group_table(n_groups, length, offsets, members):
    """A GroupTable struct over device (or, for the restatement, host) addresses of offsets and members."""
    t = GroupTable()
    t.n_groups, t.len, t.offsets, t.members = int(n_groups), int(length), offsets, members
    return t


def group_reduce(view, src_dtype, axis, table, op, center, out, scratch, stream=None):
    check(load().rb200_group_reduce(C.byref(view), src_dtype, axis, C.byref(table), op, _p(center), _p(out), _p(scratch), _p(stream)))


def group_reduce_scratch_bytes(view, axis, n_groups):
    n = int(load().rb200_group_reduce_scratch_bytes(C.byref(view), axis, n_groups))
    if n < 0:
        check(1)
    return n


def describe_group_plan(view, axis, n_groups):
    """One text line: the form, the chunk C and the split the library would reduce this view with (no device needed)."""
    lib = load()
    s = lib.rb200_describe_group_plan(C.byref(view), axis, n_groups)
    if s is None:
        check(1)
    return s.decode()


def group_plan_fields(text):
    """{key: value} of a rb200_describe_group_plan line (integers where they parse)."""
    out = {}
    for kv in text.split():
        k, v = kv.split("=", 1)
        out[k] = int(v) if v.lstrip("-").isdigit() else v
    return out


def arg_coords(origin, gstride):
    """(origin, gstride) as host int64 arrays for rb200_arg_reduce (the caller keeps them alive for the call)."""
    import numpy as np

    return np.ascontiguousarray(origin, dtype=np.int64), np.ascontiguousarray(gstride, dtype=np.int64)


def arg_reduce(view, src_dtype, axis, op, origin, gstride, out_idx, out_key, scratch, stream=None):
    """rb200_arg_reduce; origin / gstride: host int64 arrays of view.ndim entries (see arg_coords)."""
    check(load().rb200_arg_reduce(C.byref(view), src_dtype, axis, op, _p(origin.ctypes.data), _p(gstride.ctypes.data), _p(out_idx), _p(out_key),
                                  _p(scratch), _p(stream)))


def arg_reduce_scratch_bytes(view, axis):
    n = int(load().rb200_arg_reduce_scratch_bytes(C.byref(view), axis))
    if n < 0:
        check(1)
    return n


def describe_arg_plan(view, axis):
    """One text line: the form, chunk, split and CTAs the library would reduce this view with (no device needed)."""
    s = load().rb200_describe_arg_plan(C.byref(view), axis)
    if s is None:
        check(1)
    return s.decode()


def compact_count(cond, cond_dtype, run_len, counts, stream=None):
    """rb200_compact_count: counts (device int64, n_runs * chunks per run) of the selected elements of every chunk."""
    check(load().rb200_compact_count(C.byref(cond), cond_dtype, run_len, _p(counts), _p(stream)))


def compact(cond, cond_dtype, run_len, counts, incl, run_base, form, values, origin, gstride, outs, stream=None):
    """rb200_compact; values: an IndexView or None; origin / gstride: host int64 arrays or None; outs: device addresses."""
    import numpy as np

    o = np.ascontiguousarray(origin if origin is not None else np.zeros(max(cond.ndim, 1)), dtype=np.int64)
    g = np.ascontiguousarray(gstride if gstride is not None else np.zeros(max(cond.ndim, 1)), dtype=np.int64)
    ptrs = (C.c_void_p * max(len(outs), 1))(*[C.c_void_p(x) for x in outs])
    check(load().rb200_compact(C.byref(cond), cond_dtype, run_len, _p(counts), _p(incl), _p(run_base), form,
                               C.byref(values) if values is not None else None, _p(o.ctypes.data), _p(g.ctypes.data), ptrs, _p(stream)))


def describe_compact_plan(cond, run_len):
    """One text line: runs, chunks and CTAs the library would compact this condition view with (no device needed)."""
    s = load().rb200_describe_compact_plan(C.byref(cond), run_len)
    if s is None:
        check(1)
    return s.decode()


def histogram(src, src_dtype, weights, weights_dtype, table, out, bad, scratch, stream=None):
    """rb200_histogram: this view's B int64 counts (weights None) or float64 weight sums into out (device)."""
    check(load().rb200_histogram(C.byref(src), src_dtype, C.byref(weights) if weights is not None else None, weights_dtype,
                                 C.byref(table), _p(out), _p(bad), _p(scratch), _p(stream)))


def histogram_scratch_bytes(src, weighted, table):
    n = load().rb200_histogram_scratch_bytes(C.byref(src), int(bool(weighted)), C.byref(table))
    if n < 0:
        check(1)
    return n


def describe_hist_plan(src, weighted, table):
    """One text line: the form, chunk, CTAs, shared bytes and passes the library would bin this view with (no device)."""
    s = load().rb200_describe_hist_plan(C.byref(src), int(bool(weighted)), C.byref(table))
    if s is None:
        check(1)
    return s.decode()


def bin_search(src, src_dtype, sorted_ptr, n_sorted, sorted_dtype, side, out, stream=None):
    """rb200_bin_search: out[p] (device int64, the view's C order) = NumPy's searchsorted of every element."""
    check(load().rb200_bin_search(C.byref(src), src_dtype, _p(sorted_ptr), n_sorted, sorted_dtype, side, _p(out), _p(stream)))


def select_count(src, src_dtype, seg_len, state, pass_, mode, stream=None):
    """rb200_select_count: one count pass of the `pass` form over this view (or the candidate keys) into state.counts."""
    check(load().rb200_select_count(C.byref(src), src_dtype, seg_len, C.byref(state), pass_, mode, _p(stream)))


def select_choose(src, src_dtype, seg_len, state, pass_, stream=None):
    """rb200_select_choose: every target's bucket of pass pass_, on the device."""
    check(load().rb200_select_choose(C.byref(src), src_dtype, seg_len, C.byref(state), pass_, _p(stream)))


def select_rows(src, src_dtype, seg_len, targets, rank_table, skip_nan, keys, nans, stream=None):
    """rb200_select_rows: the `row` form, every target's key of every segment in one launch."""
    check(load().rb200_select_rows(C.byref(src), src_dtype, seg_len, targets, _p(rank_table), int(bool(skip_nan)), _p(keys), _p(nans),
                                   _p(stream)))


def select_scratch_bytes(src, src_dtype, seg_len, targets, segments=0):
    n = load().rb200_select_scratch_bytes(C.byref(src), src_dtype, seg_len, targets, segments)
    if n < 0:
        check(1)
    return n


def describe_select_plan(src, src_dtype, seg_len, targets, segments=0):
    """One text line: the form, digit width, passes, CTAs and buffer sizes the library would select with (no device);
    segments > 0: the view is a rank's part of that many segments (the pass form)."""
    s = load().rb200_describe_select_plan(C.byref(src), src_dtype, seg_len, targets, segments)
    if s is None:
        check(1)
    return s.decode()
