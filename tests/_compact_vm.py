"""NumPy restatement of rb200_compact_count, rb200_compact and rb200_describe_compact_plan (include/ramba_b200.h) on host
pointers.  The GPU tests compare the CUDA library against it, and the CPU tests run the engine's nonzero / flatnonzero /
extract through it, after the library's own argument checks: extend_oracle_backend() gives _oracle_backend.OracleBackend
the compact_count and compact methods that CudaBackend has."""
import numpy as np

import _index_vm

CHUNK = 4096
VALUES, FLAT, COORDS = range(3)
# rb200 dtype code -> storage (bool is stored as uint8)
NP = {0: np.float64, 1: np.float32, 2: np.int64, 3: np.int32, 4: np.uint8, 5: np.uint8, 6: np.int8, 7: np.int16, 8: np.uint16, 9: np.uint32}
_UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def _cdiv(a, b):
    return -(-a // b)


def plan(n, run_len):
    """(runs, chunks per run, runs per CTA, CTAs): the rule the library states in rb200_describe_compact_plan."""
    n_runs = n // run_len
    cpr = _cdiv(run_len, CHUNK)
    per = 1 if run_len >= CHUNK else CHUNK // run_len
    ctas = n_runs * cpr if run_len >= CHUNK else _cdiv(n_runs, per)
    return n_runs, cpr, per, ctas


def _view_array(view, dt):
    """The view as a strided numpy array of dtype dt over host memory."""
    k = view.ndim
    shape = [int(view.shape[d]) for d in range(k)]
    strides = [int(view.stride[d]) for d in range(k)]
    dt = np.dtype(dt)
    if int(np.prod(shape)) == 0:
        return np.zeros(shape, dtype=dt)
    lo = sum(min(0, (s - 1) * st) for s, st in zip(shape, strides))
    hi = sum(max(0, (s - 1) * st) for s, st in zip(shape, strides))
    mem = _index_vm._host(view.base + lo * dt.itemsize, hi - lo + 1, dt)
    return np.lib.stride_tricks.as_strided(mem[-lo:], shape, [st * dt.itemsize for st in strides])


def selected(x):
    """The selection rule on an array of stored values: x != 0 (for floats -0.0 is zero and NaN is not)."""
    return np.asarray(x).reshape(-1) != 0


def counts_of(pred, run_len):
    """counts[c * n_runs + r] of a flat C-order predicate cut into runs of run_len and chunks of CHUNK."""
    n = pred.size
    n_runs, cpr = plan(n, run_len)[:2] if n else (0, 0)
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    p = np.zeros((n_runs, cpr * CHUNK), dtype=np.int64)
    p[:, :run_len] = pred.reshape(n_runs, run_len)
    return np.ascontiguousarray(p.reshape(n_runs, cpr, CHUNK).sum(axis=2).T).reshape(-1)


def inclusive(counts, n_runs):
    """The inclusive scan of counts along each run ([cpr][n_runs] layout)."""
    if counts.size == 0:
        return counts.copy()
    return np.cumsum(counts.reshape(-1, n_runs), axis=0).reshape(-1)


def destinations(pred, run_len, counts, incl, run_base):
    """(selected positions, output position of each): run_base[r] + incl[q] - counts[q] + rank within chunk q."""
    sel = np.flatnonzero(pred).astype(np.int64)
    if sel.size == 0:
        return sel, sel
    n_runs = pred.size // run_len
    r = sel // run_len
    c = (sel - r * run_len) // CHUNK
    q = c * n_runs + r
    chunk_start = r * run_len + c * CHUNK
    rank = np.arange(sel.size, dtype=np.int64) - np.searchsorted(sel, chunk_start)
    return sel, np.asarray(run_base, dtype=np.int64)[r] + np.asarray(incl)[q] - np.asarray(counts)[q] + rank


def _pred_of(view, code):
    return selected(_view_array(view, NP[code]))


def compact_count(cond, code, run_len, counts):
    """rb200_compact_count on host pointers."""
    pred = _pred_of(cond, code)
    got = counts_of(pred, run_len)
    _index_vm._host(counts, got.size, np.int64)[:] = got


def compact(cond, code, run_len, counts, incl, run_base, form, values, origin, gstride, outs):
    """rb200_compact on host pointers."""
    pred = _pred_of(cond, code)
    shape = [int(cond.shape[d]) for d in range(cond.ndim)]
    n_runs, cpr = plan(pred.size, run_len)[:2]
    h = lambda p, n: _index_vm._host(p, n, np.int64)  # noqa: E731
    cnt, inc = h(counts, n_runs * cpr), h(incl, n_runs * cpr)
    sel, dest = destinations(pred, run_len, cnt, inc, h(run_base, n_runs))
    if sel.size == 0:
        return
    top = int(dest.max()) + 1
    if form == VALUES:
        dt = _UINT[int(values.elem_bytes)]
        _index_vm._host(outs[0], top, dt)[dest] = _view_array(values, dt).reshape(-1)[sel]
        return
    coords = np.unravel_index(sel, shape)
    if form == FLAT:
        f = np.zeros(sel.size, dtype=np.int64)
        for d in range(len(shape)):
            f += (coords[d] + int(origin[d])) * int(gstride[d])
        h(outs[0], top)[dest] = f
    else:
        for d in range(len(shape)):
            h(outs[d], top)[dest] = coords[d] + int(origin[d])


def _library_accepts(call, *args):
    """The CUDA library's validation of the same call (CPU only: it checks before it looks for a device)."""
    import torch

    from ramba_b200 import _cabi

    if torch.cuda.is_available():
        return
    _cabi.load()
    try:
        call(*args)
    except _cabi.CabiError as e:
        assert "no usable CUDA device" in str(e), "libramba_b200 would reject this compaction: %s" % e


def _oracle_compact_count(self, cond, code, run_len, counts):
    from ramba_b200 import _cabi

    _library_accepts(_cabi.compact_count, cond, code, run_len, counts)
    compact_count(cond, code, run_len, counts)


def _oracle_compact(self, cond, code, run_len, counts, incl, run_base, form, values, origin, gstride, outs):
    from ramba_b200 import _cabi

    _library_accepts(_cabi.compact, cond, code, run_len, counts, incl, run_base, form, values, origin, gstride, outs)
    compact(cond, code, run_len, counts, incl, run_base, form, values, origin, gstride, outs)


def extend_oracle_backend():
    """Let the oracle backend run compactions (through this restatement), as CudaBackend runs them on the GPU."""
    import _oracle_backend

    _oracle_backend.OracleBackend.compact_count = _oracle_compact_count
    _oracle_backend.OracleBackend.compact = _oracle_compact

