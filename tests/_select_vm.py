"""NumPy restatement of rb200_select_count, rb200_select_choose, rb200_select_rows and rb200_describe_select_plan
(include/ramba_b200.h) on host pointers.  The GPU tests compare the CUDA library against it bit for bit; the CPU tests run
the engine's median / percentile / quantile (and nan variants) through it, after the library's own argument checks:
extend_oracle_backend() gives _oracle_backend.OracleBackend the select_count, select_choose and select_rows methods that
CudaBackend has."""
import numpy as np

import _compact_vm
import _index_vm

THREADS, U, UNIT, MAX_CTAS, SHARED, ROW_HIST = 256, 4, 8192, 1056, 96 * 1024, 1024
F64, F32, I64, I32 = 0, 1, 2, 3
NP = {F64: np.float64, F32: np.float32, I64: np.int64, I32: np.int32}
READ, APPEND, CAND = range(3)


def _cdiv(a, b):
    return -(-a // b)


def keys_of(x):
    """The key map, stated once in the header: NaN (any sign / payload) -> all ones; floats: a clear sign bit set, a set
    sign bit flips every bit; ints: the sign bit flipped."""
    x = np.asarray(x)
    if x.dtype.kind == "f":
        bits = x.dtype.itemsize * 8
        u = x.view(np.uint64 if bits == 64 else np.uint32).astype(np.uint64)
        sign, full = np.uint64(1 << (bits - 1)), np.uint64((1 << bits) - 1)
        return np.where(np.isnan(x), full, np.where(u & sign, ~u & full, u | sign)).astype(np.uint64)
    bits = x.dtype.itemsize * 8
    u = x.view(np.uint64 if bits == 64 else np.uint32).astype(np.uint64)
    return u ^ np.uint64(1 << (bits - 1))


def plan(n, L, K, bits, segments=0, no_row=False):
    """The rule rb200_describe_select_plan states (shapes only)."""
    S = n // L
    GS = segments if segments > 0 else S
    kb = bits // 8
    row_bytes = ROW_HIST + L * kb
    if segments == 0 and not no_row and row_bytes <= SHARED:
        return {"form": "row", "segments": S, "all_segments": GS, "digit": 8, "passes": bits // 8, "ctas": S, "chunk": L, "rows": K,
                "groups": 1, "shared_bytes": row_bytes, "counts_bytes": 0, "scratch_bytes": 0}
    digit = 11 if GS == 1 and K <= 12 else 8
    nb = 1 << digit
    rows = min(K, SHARED // (nb * 4))
    cps = max(1, min(_cdiv(L, UNIT), _cdiv(MAX_CTAS, S))) if S else 0
    chunk = _cdiv(_cdiv(L, cps), UNIT) * UNIT if S else 0
    cps = _cdiv(L, chunk) if S else 0
    cap = min(n, max(n // 32, 65536)) if GS == 1 else 0
    return {"form": "pass", "segments": S, "all_segments": GS, "digit": digit, "passes": _cdiv(bits, digit), "ctas": S * cps, "chunk": chunk,
            "rows": rows, "groups": _cdiv(K, rows), "shared_bytes": rows * nb * 4, "counts_bytes": GS * K * nb * 8, "scratch_bytes": cap * 8}


def pass_bits(bits, digit, p):
    hi = bits - p * digit
    shift = max(hi - digit, 0)
    mask = 0 if p == 0 else ((~0) << hi) & ((1 << 64) - 1)
    return shift, hi - shift, mask


def count(keys_by_seg, st, p, bits, digit, count_nan):
    """One count pass: keys_by_seg {state row: uint64 keys}; st: dict of host arrays of the state."""
    K = st["K"]
    shift, width, mask = pass_bits(bits, digit, p)
    nb = 1 << digit
    st["counts"][:] = 0
    if p == 0:
        st["nans"][:] = 0
    full = np.uint64((1 << bits) - 1)
    for g, k in keys_by_seg.items():
        if count_nan:
            st["nans"][g] += int((k == full).sum())
        rows = 1 if p == 0 else int(st["n_slots"][g])
        for j in range(rows):
            pref = 0 if p == 0 else int(st["slot_key"][g * K + j])
            m = (k & np.uint64(mask)) == np.uint64(pref)
            d = ((k[m] >> np.uint64(shift)) & np.uint64((1 << width) - 1)).astype(np.int64)
            st["counts"][(g * K + j) * nb:(g * K + j) * nb + nb] += np.bincount(d, minlength=nb)[:nb]
    return [k[np.isin(k & np.uint64(mask), [np.uint64(st["slot_key"][g * K + j]) for j in range(int(st["n_slots"][g]))])]
            for g, k in keys_by_seg.items()] if p else None


def choose(st, p, bits, digit, off_by_one=False):
    """The choose step: each target's bucket, residual rank and key bits, then the shared count rows."""
    K, GS = st["K"], st["GS"]
    shift, width, _ = pass_bits(bits, digit, p)
    nb = 1 << digit
    for s in range(GS):
        new = []
        matched = 0
        for k in range(K):
            t = s * K + k
            row = 0 if p == 0 else int(st["slot"][t])
            h = st["counts"][(s * K + row) * nb:(s * K + row) * nb + (1 << width)]
            c = np.cumsum(h)
            r = int(st["rank"][t]) + (1 if off_by_one else 0)
            b = int(np.searchsorted(c, r, side="right"))
            b = min(b, (1 << width) - 1)
            before = int(c[b - 1]) if b else 0
            key = (0 if p == 0 else int(st["key"][t])) | (b << shift)
            st["key"][t] = np.uint64(key)
            st["rank"][t] = r - before
            if key in new:
                st["slot"][t] = new.index(key)
            else:
                st["slot"][t] = len(new)
                new.append(key)
                matched += int(h[b]) if b < h.size else 0
        st["n_slots"][s] = len(new)
        for j, key in enumerate(new):
            st["slot_key"][s * K + j] = np.uint64(key)
        st["matched"][s] = matched


def select(keys, ranks, bits, digit, off_by_one=False):
    """Every target's key of one segment's keys by the pass restatement (count + choose per digit)."""
    K = len(ranks)
    st = {"K": K, "GS": 1, "rank": np.array(ranks, np.int64), "key": np.zeros(K, np.uint64), "slot": np.zeros(K, np.int64),
          "slot_key": np.zeros(K, np.uint64), "n_slots": np.zeros(1, np.int64), "counts": np.zeros(K << digit, np.int64),
          "nans": np.zeros(1, np.int64), "matched": np.zeros(1, np.int64)}
    for p in range(_cdiv(bits, digit)):
        count({0: keys}, st, p, bits, digit, False)
        choose(st, p, bits, digit, off_by_one)
    return st["key"].copy()


def row_select(keys, ranks, bits):
    """The row form: every rank's key by 8-bit digits over the segment's keys in shared memory."""
    return select(keys, ranks, bits, 8)


# ---- on host pointers (the oracle backend) --------------------------------------------------------------------------------
def _state(st_c, digit):
    GS, K = int(st_c.segments), int(st_c.targets)
    h = _index_vm._host
    return {"K": K, "GS": GS, "rank": h(st_c.rank, GS * K, np.int64), "key": h(st_c.key, GS * K, np.uint64), "slot": h(st_c.slot, GS * K, np.int64),
            "slot_key": h(st_c.slot_key, GS * K, np.uint64), "n_slots": h(st_c.n_slots, GS, np.int64),
            "counts": h(st_c.counts, (GS * K) << digit, np.int64), "nans": h(st_c.nans, GS, np.int64), "matched": h(st_c.matched, GS, np.int64)}


def _rows_of(st_c, S):
    """The state row of each of the view's S segments."""
    if int(st_c.seg_dims) == 0:
        return np.arange(S)
    shape = [int(st_c.seg_shape[d]) for d in range(int(st_c.seg_dims))]
    g = [int(st_c.seg_gstride[d]) for d in range(int(st_c.seg_dims))]
    idx = np.indices(shape).reshape(len(shape), -1)
    return int(st_c.seg_base) + (idx * np.array(g)[:, None]).sum(axis=0)


def select_count(view, code, L, st_c, p, mode):
    from ramba_b200 import _cabi

    bits = 64 if code in (F64, I64) else 32
    n = int(np.prod([int(view.shape[d]) for d in range(int(view.ndim))]))
    f = _cabi.group_plan_fields(_cabi.describe_select_plan(view, code, L, int(st_c.targets), max(int(st_c.segments), 1)))
    digit = f["digit"]
    st = _state(st_c, digit)
    if mode == CAND:
        m = int(_index_vm._host(st_c.cand_n, 1, np.int64)[0])
        by_seg = {0: _index_vm._host(st_c.cand, m, np.uint64).copy()}
    else:
        x = _compact_vm._view_array(view, NP[code]).reshape(-1) if n else np.zeros(0, NP[code])
        S = n // L
        rows = _rows_of(st_c, S)
        by_seg = {int(rows[s]): keys_of(x[s * L:(s + 1) * L]) for s in range(S)}
    matched = count(by_seg, st, p, bits, digit, p == 0 and code in (F64, F32) and mode != CAND)
    if mode == APPEND and matched:
        m = matched[0]
        cn = _index_vm._host(st_c.cand_n, 1, np.int64)
        _index_vm._host(st_c.cand + int(cn[0]) * 8, m.size, np.uint64)[:] = m
        cn[0] += m.size


def select_choose(view, code, L, st_c, p):
    from ramba_b200 import _cabi

    bits = 64 if code in (F64, I64) else 32
    f = _cabi.group_plan_fields(_cabi.describe_select_plan(view, code, L, int(st_c.targets), max(int(st_c.segments), 1)))
    choose(_state(st_c, f["digit"]), p, bits, f["digit"])


def select_rows(view, code, L, K, rank_table, skip_nan, keys, nans):
    bits = 64 if code in (F64, I64) else 32
    x = _compact_vm._view_array(view, NP[code]).reshape(-1)
    S = x.size // L
    table = _index_vm._host(rank_table, ((L + 1) if skip_nan else 1) * K, np.int64).reshape(-1, K)
    out = _index_vm._host(keys, S * K, np.uint64)
    out_n = _index_vm._host(nans, S, np.int64)
    full = np.uint64((1 << bits) - 1)
    for s in range(S):
        k = keys_of(x[s * L:(s + 1) * L])
        c = int((k == full).sum()) if code in (F64, F32) else 0
        out_n[s] = c
        out[s * K:(s + 1) * K] = row_select(k, table[L - c if skip_nan else 0], bits)


def _library_accepts(call, *args):
    import torch

    from ramba_b200 import _cabi

    if torch.cuda.is_available():
        return
    _cabi.load()
    try:
        call(*args)
    except _cabi.CabiError as e:
        assert "no usable CUDA device" in str(e), "libramba_b200 would reject this call: %s" % e


def _oracle_select_count(self, view, code, L, st, p, mode):
    from ramba_b200 import _cabi

    _library_accepts(_cabi.select_count, view, code, L, st, p, mode)
    select_count(view, code, L, st, p, mode)


def _oracle_select_choose(self, view, code, L, st, p):
    from ramba_b200 import _cabi

    _library_accepts(_cabi.select_choose, view, code, L, st, p)
    select_choose(view, code, L, st, p)


def _oracle_select_rows(self, view, code, L, K, table, skip_nan, keys, nans):
    from ramba_b200 import _cabi

    _library_accepts(_cabi.select_rows, view, code, L, K, table, skip_nan, keys, nans)
    select_rows(view, code, L, K, table, skip_nan, keys, nans)


def extend_oracle_backend():
    """Let the oracle backend run the selection kernels (through this restatement), as CudaBackend runs them on the GPU."""
    import _oracle_backend

    _oracle_backend.OracleBackend.select_count = _oracle_select_count
    _oracle_backend.OracleBackend.select_choose = _oracle_select_choose
    _oracle_backend.OracleBackend.select_rows = _oracle_select_rows
