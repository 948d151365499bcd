"""NumPy restatement of rb200_gather, rb200_scatter and rb200_route (include/ramba_b200.h) on host pointers.  The GPU
tests compare the CUDA library against it bit for bit, and the CPU tests run the engine's integer-array indexing through
it (_oracle_backend.OracleBackend)."""
import ctypes as C

import numpy as np

_UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def _host(addr, count, dt):
    """numpy array over `count` elements of dtype `dt` at host address `addr`."""
    if count <= 0:
        return np.zeros(0, dtype=dt)
    return np.frombuffer((C.c_char * (count * np.dtype(dt).itemsize)).from_address(addr), dtype=dt)


def view_offsets(view, lin):
    """(element offsets of the entries of lin inside the view, mask of the entries in range)."""
    k = view.ndim
    shape = [int(view.shape[d]) for d in range(k)]
    stride = [int(view.stride[d]) for d in range(k)]
    size = int(np.prod(shape))
    ok = (lin >= 0) & (lin < size)
    rest = np.where(ok, lin, 0)
    off = np.zeros(len(lin), dtype=np.int64)
    for d in range(k - 1, -1, -1):
        off += (rest % shape[d]) * stride[d]
        rest //= shape[d]
    return off, ok


def _view_memory(view):
    """(numpy array over every element the view can reach, index of the view's element 0 in it)."""
    k = view.ndim
    lo = hi = 0
    for d in range(k):
        reach = max(int(view.shape[d]) - 1, 0) * int(view.stride[d])
        lo, hi = (lo + reach, hi) if reach < 0 else (lo, hi + reach)
    eb = view.elem_bytes
    return _host(view.base + lo * eb, hi - lo + 1, _UINT[eb]), -lo


def gather(view, lin_ptr, n, out_ptr, bad_ptr):
    if n == 0:
        return
    lin = _host(lin_ptr, n, np.int64)
    off, ok = view_offsets(view, lin)
    out = _host(out_ptr, n, _UINT[view.elem_bytes])
    if int(np.prod([view.shape[d] for d in range(view.ndim)])) > 0:
        mem, o0 = _view_memory(view)
        out[ok] = mem[off[ok] + o0]
    out[~ok] = 0
    _host(bad_ptr, 1, np.uint64)[0] += np.uint64((~ok).sum())


def scatter(view, lin_ptr, n, values_ptr, bad_ptr):
    if n == 0:
        return
    lin = _host(lin_ptr, n, np.int64)
    off, ok = view_offsets(view, lin)
    vals = _host(values_ptr, n, _UINT[view.elem_bytes])
    if ok.any():
        mem, o0 = _view_memory(view)
        mem[off[ok] + o0] = vals[ok]
    _host(bad_ptr, 1, np.uint64)[0] += np.uint64((~ok).sum())


def locate(table, lin):
    """(owner, owner's local element offset) of every entry of lin (owner -1: out of range)."""
    k = table.ndim
    shape = [int(table.shape[d]) for d in range(k)]
    n_cells = [int(table.n_cells[d]) for d in range(k)]
    total_cells = int(np.prod(n_cells))
    cuts_all = _host(table.cuts, max(int(table.cut_start[d]) + n_cells[d] + 1 for d in range(k)), np.int64)
    owners = _host(table.cell_owner, total_cells, np.int32)
    offsets = _host(table.cell_offset, total_cells, np.int64)
    strides = _host(table.cell_stride, total_cells * k, np.int64).reshape(total_cells, k)
    size = int(np.prod(shape))
    ok = (lin >= 0) & (lin < size)
    rest = np.where(ok, lin, 0)
    coords = []
    for d in range(k - 1, -1, -1):
        coords.append(rest % shape[d])
        rest = rest // shape[d]
    coords = coords[::-1]
    cell = np.zeros(len(lin), dtype=np.int64)
    los = []
    for d in range(k):
        cut = cuts_all[int(table.cut_start[d]):int(table.cut_start[d]) + n_cells[d] + 1]
        j = np.searchsorted(cut, coords[d], side="right") - 1
        los.append(cut[j])
        cell = cell * n_cells[d] + j
    off = offsets[cell].copy()
    for d in range(k):
        off += (coords[d] - los[d]) * strides[cell, d]
    owner = np.where(ok, owners[cell], -1).astype(np.int64)
    return owner, off


def route(table, lin_ptr, n, offsets_ptr, slots_ptr, counts_ptr, bad_ptr):
    R = int(table.n_ranks)
    counts = _host(counts_ptr, R, np.int64)
    if n == 0:
        counts[:] = 0
        return
    lin = _host(lin_ptr, n, np.int64)
    owner, off = locate(table, lin)
    valid = owner >= 0
    cnt = np.bincount(owner[valid], minlength=R).astype(np.int64)
    counts[:] = cnt
    order = np.argsort(np.where(valid, owner, R), kind="stable")  # grouped by owner, in the order of i inside a group
    slot = np.full(n, -1, dtype=np.int64)
    nv = int(valid.sum())
    slot[order[:nv]] = np.arange(nv, dtype=np.int64)
    _host(slots_ptr, n, np.int64)[:] = slot
    if nv:
        _host(offsets_ptr, nv, np.int64)[:] = off[order[:nv]]
    _host(bad_ptr, 1, np.uint64)[0] += np.uint64(n - nv)

