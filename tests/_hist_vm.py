"""NumPy restatement of rb200_histogram, rb200_bin_search and rb200_describe_hist_plan (include/ramba_b200.h) on host
pointers.  The GPU tests compare the CUDA library against it bit for bit (weighted sums included: the restatement adds
in the library's fold order), and the CPU tests run the engine's histogram / bincount / searchsorted / digitize through
it, after the library's own argument checks: extend_oracle_backend() gives _oracle_backend.OracleBackend the histogram
and bin_search methods that CudaBackend has."""
import numpy as np

import _compact_vm
import _index_vm

THREADS, WARPS, U = 256, 8, 4
UNIT, MAX_CTAS, SHARED = 8192, 1056, 96 * 1024
UNIFORM, EDGES, INTEGER = range(3)
F64, F32, I64, I32 = 0, 1, 2, 3
NP = {F64: np.float64, F32: np.float32, I64: np.int64, I32: np.int32}


def _cdiv(a, b):
    return -(-a // b)


def plan(n, B, weighted, table_bytes, elem_bytes=8):
    """The rule rb200_describe_hist_plan states: {form, chunk, ctas, passes, slab, shared_bytes, table, scratch}."""
    ctas = min(_cdiv(n, UNIT), MAX_CTAS) if n else 0
    chunk = _cdiv(_cdiv(n, ctas), UNIT) * UNIT if n else 0
    ctas = _cdiv(n, chunk) if n else 0
    if not weighted:
        form = "shared" if B * 4 <= SHARED else "global"
        slab = B if form == "shared" else 0
        rows = slab * 4
    else:
        fit = (SHARED - WARPS * 32 * 8) // (WARPS * 8)
        form = "shared" if B <= fit else "slab"
        slab = min(B, fit)
        rows = (WARPS * slab + WARPS * 32) * 8
    passes = _cdiv(B, slab) if weighted else 1
    toff = _cdiv(rows, 16) * 16
    tshared = table_bytes > 0 and toff + table_bytes <= SHARED
    shared = 0 if form == "global" and not tshared else toff + (table_bytes if tshared else 0)
    return {"form": form, "chunk": chunk, "ctas": ctas, "passes": passes, "slab": slab, "shared_bytes": shared,
            "table": "none" if table_bytes == 0 else ("shared" if tshared else "global"), "scratch": ctas * slab * 8 if weighted else 0}


def _lt_nan(a, b):
    """NumPy's sort order a < b (NaN after every number), elementwise."""
    with np.errstate(invalid="ignore"):
        if np.asarray(a).dtype.kind == "f" or np.asarray(b).dtype.kind == "f":
            return (a < b) | ((b != b) & (a == a))
        return a < b


def _bound(x, dt, f, i, ge):
    if dt == I64:
        v, b = x.astype(np.int64), np.int64(i)
    else:
        v, b = x.astype(NP[dt]), NP[dt](f)
    with np.errstate(invalid="ignore"):
        return v >= b if ge else v <= b


def bins_of(x, t, edges):
    """Every element's bin under table t: -1 dropped, -2 bad (the kernel's rule, vectorised)."""
    B = int(t["n_bins"])
    if t["form"] == INTEGER:
        v = x.astype(np.int64)
        return np.where((v < 0) | (v >= B), -2, v)
    if t["form"] == EDGES:
        c = x.astype(NP[t["edge_dtype"]])
        j = np.searchsorted(edges[:B], c, side="right").astype(np.int64)
        last = np.where(_lt_nan(edges[B], c), -1, B - 1)
        return np.where(j == 0, -1, np.where(j < B, j - 1, last))
    keep = _bound(x, t["lo_dtype"], t["lo"], t["lo_i"], True) & _bound(x, t["hi_dtype"], t["hi"], t["hi_i"], False)
    E, S, D = NP[t["edge_dtype"]], NP[t["sub_dtype"]], NP[t["div_dtype"]]
    xe = x.astype(E)
    with np.errstate(all="ignore"):
        s = xe.astype(S) - S(t["first"])
        q = (s.astype(D) / D(t["denom"])) * D(B)
        q = np.where(np.isfinite(q) & (np.abs(q) < 2.0 ** 62), q, -1e300)
        idx = np.trunc(q).clip(-(2 ** 62), 2 ** 62).astype(np.int64)
    idx = np.where(idx == B, B - 1, idx)
    out = (idx < 0) | (idx >= B)
    i0 = np.clip(idx, 0, B - 1)
    idx = np.where(xe < edges[i0], idx - 1, idx)
    i1 = np.clip(idx + 1, 0, B)
    idx = np.where((idx != B - 1) & (xe >= edges[i1]), idx + 1, idx)
    res = np.where(out | (idx < 0), -2, idx)
    return np.where(keep, res, -1)


def positions(n, chunk, eb):
    """(cta, warp, slot order inside the warp, lane) of C-order positions 0..n-1 (the kernel's walk)."""
    E = 16 // eb
    p = np.arange(n, dtype=np.int64)
    c = p // chunk
    r = p - c * chunk
    step, q = np.divmod(r, THREADS * E * U)
    w, q2 = np.divmod(q, 32 * E * U)
    k, q3 = np.divmod(q2, 32 * E)
    lane, u = np.divmod(q3, E)
    return c, w, (step * U + k) * E + u, lane


def weighted_sums(bins, wts, n, B, chunk, ctas, eb):
    """B float64 sums in the library's fold order: per (CTA, warp, slot) the lanes of one bin in lane order, those sums
    into the warp's row in slot order, rows in warp order from +0.0, CTAs in CTA order from +0.0."""
    c, w, slot, lane = positions(n, chunk, eb)
    m = bins >= 0
    c, w, slot, lane, b, v = c[m], w[m], slot[m], lane[m], bins[m], wts[m]
    out = np.zeros(B, dtype=np.float64)
    if not b.size:
        return out
    with np.errstate(all="ignore"):
        # groups (cta, warp, slot, bin), members in lane order
        order = np.lexsort((lane, b, slot, w, c))
        key = np.stack([c[order], w[order], slot[order], b[order]])
        new = np.ones(order.size, dtype=bool)
        new[1:] = (key[:, 1:] != key[:, :-1]).any(axis=0)
        gid = np.cumsum(new) - 1
        gsum = np.zeros(int(gid[-1]) + 1, dtype=np.float64)
        np.add.at(gsum, gid, v[order])
        gc, gw, gslot, gb = key[:, new]
        # into the warp rows in slot order
        rows = np.zeros((ctas, WARPS, B), dtype=np.float64)
        o2 = np.lexsort((gslot, gb, gw, gc))
        np.add.at(rows.reshape(-1), ((gc * WARPS + gw) * B + gb)[o2], gsum[o2])
        cta = np.zeros((ctas, B), dtype=np.float64)
        for i in range(WARPS):
            cta += rows[:, i, :]
        for i in range(ctas):
            out += cta[i]
    return out


def _table_dict(tb):
    return {f: getattr(tb, f) for f, _ in tb._fields_}


def histogram(src, src_code, wview, w_code, table, out, bad):
    """rb200_histogram on host pointers."""
    t = _table_dict(table)
    B = int(t["n_bins"])
    x = _compact_vm._view_array(src, NP[src_code]).reshape(-1)
    edges = None
    if t["form"] != INTEGER:
        edges = _index_vm._host(t["edges"], B + 1, NP[t["edge_dtype"]])
    bins = bins_of(x, t, edges)
    n_bad = int((bins == -2).sum())
    bins = np.where(bins == -2, -1, bins)
    if n_bad:
        _index_vm._host(bad, 1, np.int64)[0] += n_bad
    if wview is None:
        _index_vm._host(out, B, np.int64)[:] = np.bincount(bins[bins >= 0], minlength=B)[:B]
        return
    wts = _compact_vm._view_array(wview, NP[w_code]).reshape(-1).astype(np.float64)
    P = plan(x.size, B, True, 0)
    _index_vm._host(out, B, np.float64)[:] = weighted_sums(bins, wts, x.size, B, P["chunk"], P["ctas"], x.dtype.itemsize)


def bin_search(src, src_code, sorted_ptr, n_sorted, sorted_code, side, out):
    """rb200_bin_search on host pointers."""
    x = _compact_vm._view_array(src, NP[src_code]).reshape(-1)
    tab = _index_vm._host(sorted_ptr, n_sorted, NP[sorted_code])
    _index_vm._host(out, x.size, np.int64)[:] = np.searchsorted(tab, x.astype(NP[sorted_code]), side="right" if side else "left")


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
        assert "no usable CUDA device" in str(e), "libramba_b200 would reject this call: %s" % e


def _oracle_histogram(self, view, src_code, wview, w_code, table, out, bad):
    from ramba_b200 import _cabi

    _library_accepts(_cabi.histogram, view, src_code, wview, w_code, table, out, bad, 0x1000)
    histogram(view, src_code, wview, w_code, table, out, bad)
    return None


def _oracle_bin_search(self, view, src_code, sorted_ptr, n_sorted, sorted_code, side, out):
    from ramba_b200 import _cabi

    _library_accepts(_cabi.bin_search, view, src_code, sorted_ptr, n_sorted, sorted_code, side, out)
    bin_search(view, src_code, sorted_ptr, n_sorted, sorted_code, side, out)


def extend_oracle_backend():
    """Let the oracle backend run the binning kernels (through this restatement), as CudaBackend runs them on the GPU."""
    import _oracle_backend

    _oracle_backend.OracleBackend.histogram = _oracle_histogram
    _oracle_backend.OracleBackend.bin_search = _oracle_bin_search
