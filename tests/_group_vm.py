"""NumPy restatement of rb200_group_reduce and rb200_describe_group_plan (include/ramba_b200.h) on host pointers.  The GPU
tests compare the CUDA library against it bit for bit, and the CPU tests run the engine's groupby through it
(_oracle_backend.OracleBackend)."""
import ctypes as C

import numpy as np

import _index_vm

SUM, PROD, MIN, MAX, NANSUM, NANCOUNT, SQDEV = range(7)
_NP = {0: np.float64, 1: np.float32, 2: np.int64, 3: np.int32}  # rb200 dtype code -> storage
PLAN_SMS = 132
TARGET_CTAS = 4 * PLAN_SMS
MIN_CHUNK = 1024
MAX_SPLIT = 1024
ROW_MAX_GROUPS = 1024


def _cdiv(a, b):
    return -(-a // b)


def plan(shape, strides, axis, G):
    """(form, chunk C) of the view: the rule the library states in rb200_describe_group_plan."""
    k = len(shape)
    L, sa = int(shape[axis]), int(strides[axis])
    kept = []
    O = I = 1
    n_outer = 0
    for side, (d0, d1) in enumerate(((0, axis), (axis + 1, k))):
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
    if I == 1 and sa == 1 and G <= ROW_MAX_GROUPS:
        form = "row"
    elif len(inner) == 1 and inner[0][1] == 1 and inner[0][0] >= 32:
        form = "column"
    else:
        form = "general"
    if form == "row":
        K = 1
        if O < TARGET_CTAS and L >= 2 * MIN_CHUNK:
            K = min(_cdiv(TARGET_CTAS, max(O, 1)), L // MIN_CHUNK)
        if K <= 1:
            ncl = min(min(64, _cdiv(256, G)), max(L, 1))
            C_ = max(_cdiv(L, ncl), 1)
        else:
            C_ = _cdiv(L, K)
    else:
        base = _cdiv(O * I, 256) * G
        S = 1
        if base < TARGET_CTAS and L >= 2 * MIN_CHUNK:
            S = min(_cdiv(TARGET_CTAS, max(base, 1)), L // MIN_CHUNK, MAX_SPLIT)
        C_ = max(_cdiv(L, S), 1)
    return form, C_


def _host(addr, count, dt):
    return _index_vm._host(addr, count, dt)


def _source(view, src_code):
    """The view as a strided numpy array over host memory."""
    k = view.ndim
    shape = [int(view.shape[d]) for d in range(k)]
    strides = [int(view.stride[d]) for d in range(k)]
    dt = np.dtype(_NP[src_code])
    if int(np.prod(shape)) == 0:
        return np.zeros(shape, dtype=dt)
    lo = sum(min(0, (s - 1) * st) for s, st in zip(shape, strides))
    hi = sum(max(0, (s - 1) * st) for s, st in zip(shape, strides))
    mem = _host(view.base + lo * dt.itemsize, hi - lo + 1, dt)
    return np.lib.stride_tricks.as_strided(mem[-lo:], shape, [st * dt.itemsize for st in strides])


def identity(op, is_float):
    if op == PROD:
        return 1
    if op == MIN:
        return np.inf if is_float else np.iinfo(np.int64).max
    if op == MAX:
        return -np.inf if is_float else np.iinfo(np.int64).min
    return 0


def _combine(op, a, b):
    if op == PROD:
        return a * b
    if op == MIN:
        return np.where(b < a, b, a)
    if op == MAX:
        return np.where(b > a, b, a)
    return a + b


def _step(op, acc, x, c, src_float):
    if op == SQDEV:
        d = x.astype(np.float64) - c
        return acc + d * d
    if op == NANCOUNT:
        return np.where(np.isnan(x), acc, acc + 1) if src_float else acc + 1
    if op == NANSUM:
        return np.where(np.isnan(x), acc, acc + x.astype(acc.dtype)) if src_float else acc + x.astype(acc.dtype)
    return _combine(op, acc, x.astype(acc.dtype))


def reduce(x, axis, labels, G, op, C_, center=None):
    """out[o, g, i] as (O, G, I) in the accumulator class: chunks of C_ positions, each folded in ascending order from the
    identity, the chunk partials folded in chunk order from the identity."""
    src_float = x.dtype.kind == "f"
    acc_dt = np.float64 if (src_float or op == SQDEV) else np.int64
    L = x.shape[axis]
    O = int(np.prod(x.shape[:axis]))
    I = int(np.prod(x.shape[axis + 1:]))
    x3 = np.ascontiguousarray(x).reshape(O, L, I)
    cen = None if center is None else np.asarray(center, dtype=np.float64).reshape(O, G, I)
    ident = np.array(identity(op, acc_dt == np.float64), dtype=acc_dt)
    with np.errstate(all="ignore"):
        out = np.full((O, G, I), ident, dtype=acc_dt)
        for s0 in range(0, max(L, 1), C_):
            part = np.full((O, G, I), ident, dtype=acc_dt)
            for t in range(s0, min(L, s0 + C_)):
                g = labels[t]
                part[:, g, :] = _step(op, part[:, g, :], x3[:, t, :], None if cen is None else cen[:, g, :], src_float)
            out = _combine(op, out, part)
    return out


def group_reduce(view, src_code, axis, table, op, center_ptr, out_ptr):
    """rb200_group_reduce on host pointers."""
    x = _source(view, src_code)
    G, L = int(table.n_groups), int(table.len)
    assert L == x.shape[axis]
    offs = _host(table.offsets, G + 1, np.int64)
    mem = _host(table.members, L, np.int64)
    labels = np.zeros(L, dtype=np.int64)
    for g in range(G):
        labels[mem[offs[g]:offs[g + 1]]] = g
    shape = [int(view.shape[d]) for d in range(view.ndim)]
    strides = [int(view.stride[d]) for d in range(view.ndim)]
    _, C_ = plan(shape, strides, axis, G)
    n_out = int(np.prod(shape[:axis] + shape[axis + 1:])) * G
    center = _host(center_ptr, n_out, np.float64) if op == SQDEV else None
    res = reduce(x, axis, labels, G, op, C_, center)
    acc_dt = res.dtype
    _host(out_ptr, res.size, acc_dt)[:] = res.reshape(-1)


def _library_accepts(view, src_code, axis, table, op, center, out):
    """The CUDA library's validation of the same call (CPU only: it checks before it looks for a device)."""
    import torch

    from ramba_b200 import _cabi

    if torch.cuda.is_available():
        return
    lib = _cabi.load()
    rc = lib.rb200_group_reduce(C.byref(view), src_code, axis, C.byref(table), op, C.c_void_p(center) if center else None,
                                C.c_void_p(out) if out else None, C.c_void_p(1), None)
    msg = lib.rb200_last_error().decode() if rc else ""
    assert rc == 0 or "no usable CUDA device" in msg, "libramba_b200 would reject this grouped reduction: " + msg

