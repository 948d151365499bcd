"""NumPy restatement of rb200_arg_reduce and rb200_describe_arg_plan (include/ramba_b200.h) on host pointers.  The GPU
tests compare the CUDA library against it, and the CPU tests run the engine's argmax / argmin / nanargmax / nanargmin
through it, after the library's own argument checks: extend_oracle_backend() gives _oracle_backend.OracleBackend the
arg_reduce method that CudaBackend has."""
import ctypes as C

import numpy as np

import _group_vm

ARG_MAX, ARG_MIN, ARG_NANMAX, ARG_NANMIN = range(4)
ALL_AXES = -1
NO_INDEX = np.iinfo(np.int64).max
KEY_MIN = np.iinfo(np.int64).min
PLAN_SMS = 132
TARGET_CTAS = 8 * PLAN_SMS
MIN_CHUNK = 1024
MAX_SPLIT = 1024
CHUNK_ALIGN = 64


def _cdiv(a, b):
    return -(-a // b)


def plan(shape, strides, axis):
    """(form, chunk, split) of the view: the rule the library states in rb200_describe_arg_plan."""
    if axis == ALL_AXES:
        n = int(np.prod(shape))
        ctas = max(1, min(TARGET_CTAS, _cdiv(n, 256 * 16)))
        chunk = max(_cdiv(_cdiv(n, ctas), CHUNK_ALIGN) * CHUNK_ALIGN, CHUNK_ALIGN)
        return "global", chunk, max(_cdiv(n, chunk), 1)
    L, sa = int(shape[axis]), int(strides[axis])
    kept = []
    O = I = 1
    n_outer = 0
    for side, (d0, d1) in enumerate(((0, axis), (axis + 1, len(shape)))):
        first = len(kept)
        for d in range(d0, d1):
            if side == 0:
                O *= int(shape[d])
            else:
                I *= int(shape[d])
            if shape[d] == 1:
                continue
            if len(kept) > first and kept[-1][1] == strides[d] * shape[d]:
                kept[-1] = [kept[-1][0] * int(shape[d]), int(strides[d])]
                continue
            kept.append([int(shape[d]), int(strides[d])])
        if side == 0:
            n_outer = len(kept)
    inner = kept[n_outer:]
    if I == 1 and sa == 1:
        form = "row"
    elif len(inner) == 1 and inner[0][1] == 1 and inner[0][0] >= 32:
        form = "column"
    else:
        form = "general"
    base = _cdiv(O * I, 8 if form == "row" else 256)
    S = 1
    if base < TARGET_CTAS and L >= 2 * MIN_CHUNK:
        S = min(_cdiv(TARGET_CTAS, max(base, 1)), L // MIN_CHUNK, MAX_SPLIT)
    chunk = _cdiv(_cdiv(L, S), CHUNK_ALIGN) * CHUNK_ALIGN if S > 1 else max(L, 1)
    return form, chunk, max(_cdiv(L, chunk), 1)


def keys(x, op):
    """(order key, has a candidate) of every element of x, as int64 / bool arrays of x's shape."""
    x = np.asarray(x)
    ok = np.ones(x.shape, dtype=bool)
    if x.dtype.kind == "f":
        ibits = x.view(np.int64 if x.dtype.itemsize == 8 else np.int32).astype(np.int64)
        ibits = np.where(x == 0, 0, ibits)
        k = np.where(ibits >= 0, ibits, ibits ^ NO_INDEX)
        nan = np.isnan(x)
        k = np.where(nan, KEY_MIN if op == ARG_MIN else NO_INDEX, k)
        if op in (ARG_NANMAX, ARG_NANMIN):
            ok = ~nan
    else:
        k = x.astype(np.int64)
    if op in (ARG_MIN, ARG_NANMIN):
        k = ~k
    return k.astype(np.int64), ok


def reduce(x, axis, op, origin, gstride):
    """(index, key) per output of view x (an array), with x's element c at global coordinate origin + c of an array with
    C-order strides gstride: flat indices over every axis (axis = ALL_AXES), positions along `axis` otherwise."""
    k, ok = keys(x, op)
    k = np.where(ok, k, KEY_MIN)
    if axis == ALL_AXES:
        coords = np.indices(x.shape, dtype=np.int64) if x.ndim else np.zeros((0,), np.int64)
        g = np.zeros(x.shape, dtype=np.int64)
        for d in range(x.ndim):
            g += (coords[d] + int(origin[d])) * int(gstride[d])
        kf, gf = k.reshape(1, -1), np.where(ok, g, NO_INDEX).reshape(1, -1)
        out_shape = ()
    else:
        pos = np.arange(x.shape[axis], dtype=np.int64) + int(origin[axis])
        g = np.broadcast_to(pos.reshape([-1 if d == axis else 1 for d in range(x.ndim)]), x.shape)
        kf = np.moveaxis(k, axis, -1).reshape(-1, x.shape[axis])
        gf = np.moveaxis(np.where(ok, g, NO_INDEX), axis, -1).reshape(-1, x.shape[axis])
        out_shape = x.shape[:axis] + x.shape[axis + 1:]
    n = kf.shape[0]
    best_k = np.full(n, KEY_MIN, dtype=np.int64)
    best_i = np.full(n, NO_INDEX, dtype=np.int64)
    if kf.shape[1]:
        best_k = kf.max(axis=1)
        best_i = np.where(kf == best_k[:, None], gf, NO_INDEX).min(axis=1)
    return best_i.reshape(out_shape), best_k.reshape(out_shape)


def arg_reduce(view, src_code, axis, op, origin, gstride, out_idx, out_key):
    """rb200_arg_reduce on host pointers."""
    x = _group_vm._source(view, src_code)
    idx, key = reduce(x, axis, op, origin, gstride)
    _group_vm._host(out_idx, max(idx.size, 1), np.int64)[:idx.size] = idx.reshape(-1)
    _group_vm._host(out_key, max(key.size, 1), np.int64)[:key.size] = key.reshape(-1)


def _library_accepts(view, src_code, axis, op, origin, gstride, out_idx, out_key):
    """The CUDA library's validation of the same call (CPU only: it checks before it looks for a device)."""
    import torch

    from ramba_b200 import _cabi

    if torch.cuda.is_available():
        return
    lib = _cabi.load()
    o, g = _cabi.arg_coords(origin, gstride)
    rc = lib.rb200_arg_reduce(C.byref(view), src_code, axis, op, o.ctypes.data, g.ctypes.data, C.c_void_p(out_idx) if out_idx else None,
                              C.c_void_p(out_key) if out_key else None, C.c_void_p(1), None)
    msg = lib.rb200_last_error().decode() if rc else ""
    assert rc == 0 or "no usable CUDA device" in msg, "libramba_b200 would reject this index reduction: " + msg


def _oracle_arg_reduce(self, view, src_code, axis, op, origin, gstride, out_idx, out_key):
    """OracleBackend.arg_reduce: the library's argument checks, then the restatement on host buffers."""
    _library_accepts(view, src_code, axis, op, origin, gstride, out_idx, out_key)
    arg_reduce(view, src_code, axis, op, origin, gstride, out_idx, out_key)
    return None


def extend_oracle_backend():
    """Let the oracle backend run index reductions (through this restatement), as CudaBackend runs them on the GPU."""
    import _oracle_backend

    _oracle_backend.OracleBackend.arg_reduce = _oracle_arg_reduce
