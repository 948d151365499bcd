"""Order statistics: median, nanmedian, percentile, nanpercentile, quantile and nanquantile.

CPU: the engine through the NumPy restatement of the kernels (_select_vm) against NumPy with == and the same dtype and
shape, for every function, method and stored dtype, 0-d to 4-d, every axis, keepdims, scalar / 1-D / 2-D q, view kinds,
lazy inputs and both DAG modes; edge data (n = 1 and 2, all equal, last-bit neighbours, keys straddling every digit
boundary, signed zeros, infinities, subnormals, NaN anywhere, int64 extremes and values near 2^53, float32 values near
FLT_MAX) and NumPy's errors and warnings; the restatement against a brute-force sort, each check shown to reject a wrong
restatement; the plan, the argument checks and the exports of the C-ABI; no spills; gloo worlds 2, 3, 4 and 8 against
world 1 and NumPy, with the transfer counters.
GPU: every kernel against the restatement bit for bit in each form and dtype, the public functions against NumPy at the
benchmark's scale, a float32 selection over more than 2^31 elements in one bucket, and world 2 over NCCL where two GPUs
exist."""
import ctypes as C
import os
import re
import socket
import subprocess
import sys
import types
import warnings

import numpy as onp
import pytest

import _select_vm as SV

HERE = os.path.dirname(os.path.abspath(__file__))
SV.extend_oracle_backend()  # (also for the oracle stand-in of the -m gpu tests under RB200_DRY_GPU_TESTS)
DTYPES = (onp.float64, onp.float32, onp.int64, onp.int32, onp.int16, onp.int8, onp.uint8, onp.uint16, onp.uint32, onp.bool_)
SHAPES = [(), (1,), (2,), (7,), (5, 9), (3, 4, 5), (2, 3, 4, 5)]
METHODS = ("inverted_cdf", "averaged_inverted_cdf", "closest_observation", "interpolated_inverted_cdf", "hazen", "weibull", "linear",
           "median_unbiased", "normal_unbiased", "lower", "higher", "midpoint", "nearest")
FUNCS = ("median", "nanmedian", "percentile", "nanpercentile", "quantile", "nanquantile")


@pytest.fixture
def q_engine():
    import _oracle_backend
    from ramba_b200 import ramba
    from ramba_b200.runtime import RT

    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()
    _oracle_backend.install()
    yield
    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()


def _data(shape, dtype, seed, nan=0.0):
    r = onp.random.default_rng(seed)
    dt = onp.dtype(dtype)
    if dt.kind == "f":
        x = onp.asarray((r.standard_normal(shape) * 10).astype(dt))
        if nan:
            x[onp.asarray(r.random(shape) < nan)] = onp.nan
        return x
    if dt == onp.bool_:
        return r.random(shape) < 0.5
    info = onp.iinfo(dt)
    return r.integers(max(info.min, -100), min(info.max, 100), size=shape, endpoint=True).astype(dt)


def _call(mod, name, x, q=None, **kw):
    f = getattr(mod, name)
    return f(x, **kw) if name.endswith("median") else f(x, q, **kw)


def _same(got, exp, what):
    """got (a ramba array or a NumPy scalar) == exp with NumPy's dtype and shape (NaN equal to NaN)."""
    from ramba_b200 import ndarray

    e = onp.asarray(exp)
    if isinstance(got, ndarray):
        assert e.ndim > 0 or not isinstance(exp, onp.generic), (what, "NumPy gives a scalar")
        g = got.asarray()
    else:
        assert isinstance(got, onp.generic) and isinstance(exp, onp.generic), (what, type(got), type(exp))
        g = onp.asarray(got)
    assert g.dtype == e.dtype and g.shape == e.shape, (what, g.dtype, e.dtype, g.shape, e.shape)
    assert onp.array_equal(g, e, equal_nan=e.dtype.kind == "f"), (what, g, e)


def _check(rb, name, x, X, q=None, **kw):
    with warnings.catch_warnings(record=True) as we:
        warnings.simplefilter("always")
        try:
            exp = _call(onp, name, x, q, **kw)
        except Exception as ex:  # NumPy's exception class
            with pytest.raises(type(ex)):
                _call(rb, name, X, q, **kw)
            return
    with warnings.catch_warnings(record=True) as wg:
        warnings.simplefilter("always")
        got = _call(rb, name, X, q, **kw)
    _same(got, exp, (name, x.dtype, x.shape, q, kw))
    ew = {w.category for w in we if w.category is RuntimeWarning}
    gw = {w.category for w in wg if w.category is RuntimeWarning}
    assert ew == gw, (name, x.dtype, x.shape, kw, [str(w.message) for w in we], [str(w.message) for w in wg])


def _q_for(name, q):
    return None if name.endswith("median") else (q * 100 if "percentile" in name else q)


# ---- every function, dtype, rank, axis -------------------------------------------------------------------------------------
def _check_dtypes_and_ranks(rb):
    for shape in SHAPES:
        for dt in DTYPES:
            x = _data(shape, dt, 3, nan=0.1)
            X = rb.fromarray(x)
            x = x.astype(X.dtype)  # (fromarray keeps a 0-d value in its default dtype)
            axes = [None] + list(range(-len(shape), len(shape)))
            for ax in axes:
                for name in FUNCS:
                    _check(rb, name, x, X, _q_for(name, 0.3), axis=ax)
                    if ax is not None and ax % 2:
                        _check(rb, name, x, X, _q_for(name, onp.array([0.0, 0.25, 1.0])), axis=ax, keepdims=True)


def test_every_dtype_and_rank(q_engine):
    import ramba_b200 as rb

    _check_dtypes_and_ranks(rb)


def _check_methods_and_q(rb):
    x = _data((6, 11), onp.float64, 4, nan=0.05)
    xi = _data((6, 11), onp.int32, 4)
    xf = _data((37,), onp.float32, 5)
    qs = [0.5, onp.float32(0.35), [0.0, 0.1, 0.5, 0.9, 1.0], onp.array([[0.2, 0.7], [1.0, 0.0]]), onp.linspace(0, 1, 21)]
    for m in METHODS:
        for q in qs:
            for arr in (x, xi, xf):
                X = rb.fromarray(arr)
                for name in ("quantile", "nanquantile", "percentile", "nanpercentile"):
                    qq = onp.asarray(q) * 100 if "percentile" in name else q
                    _check(rb, name, arr, X, qq, axis=None, method=m)
                    _check(rb, name, arr, X, qq, axis=-1, method=m)
    X = rb.fromarray(x)
    _check(rb, "quantile", x, X, rb.fromarray(onp.array([0.25, 0.75])), axis=0)


def test_every_method_and_q(q_engine):
    import ramba_b200 as rb

    _check_methods_and_q(rb)


VIEWS = [
    lambda a: a[1:, ::2], lambda a: a[::-1], lambda a: a.T, lambda a: a[:, 3], lambda a: a[2:7, ::-3],
]


def _check_views(rb):
    x = _data((9, 13), onp.float64, 6, nan=0.1)
    X = rb.fromarray(x)
    for v in VIEWS:
        for name in FUNCS:
            for ax in (None, 0, -1):
                if v(x).ndim == 1 and ax not in (None, 0, -1):
                    continue
                _check(rb, name, v(x), v(X), _q_for(name, 0.4), axis=ax)
    b = onp.broadcast_to(x[:1], (5, 13))
    _check(rb, "median", b, rb.broadcast_to(X[:1], (5, 13)), axis=0)
    lazy = X * 2.0 + 1.0
    _check(rb, "quantile", x * 2.0 + 1.0, lazy, 0.3, axis=1)
    _check(rb, "median", x * 2.0 + 1.0, X * 2.0 + 1.0)


def test_views_and_lazy_inputs(q_engine):
    import ramba_b200 as rb

    _check_views(rb)


def test_without_the_dag(q_engine, monkeypatch):
    import ramba_b200 as rb
    from ramba_b200 import ramba

    monkeypatch.setattr(ramba, "RAMBA_NO_DAG", True, raising=False)
    x = _data((6, 7), onp.float32, 7, nan=0.2)
    X = rb.fromarray(x) + 0.5
    for name in FUNCS:
        _check(rb, name, x + onp.float32(0.5), X, _q_for(name, 0.6), axis=1)


# ---- edge data ---------------------------------------------------------------------------------------------------------------
def _edge_cases():
    f64, f32 = onp.float64, onp.float32
    tiny = onp.finfo(f64).smallest_subnormal
    yield onp.array([3.5])
    yield onp.array([3.5, -1.0])
    yield onp.full(33, 2.25)
    yield onp.array([1.0, onp.nextafter(1.0, 2.0)] * 5)
    yield onp.array([-0.0, 0.0, -0.0, 1.0, -1.0])
    yield onp.array([onp.inf, -onp.inf, 0.0, onp.inf, 5.0, -onp.inf])
    yield onp.array([tiny, -tiny, 2 * tiny, 0.0, -3 * tiny])
    yield onp.array([onp.nan, 1.0, 2.0, 3.0])
    yield onp.array([1.0, 2.0, 3.0, onp.nan])
    yield onp.array([1.0, onp.nan, 3.0, 2.0, 0.5])
    yield onp.full(6, onp.nan)
    yield onp.array([-onp.nan, 2.0, 1.0])
    # keys straddling every digit boundary: values whose bit patterns differ at bit 8k, 11k
    base = onp.array([1.0]).view(onp.uint64)[0]
    yield onp.array([base + onp.uint64(1 << b) for b in range(0, 52)] + [base], dtype=onp.uint64).view(f64)
    yield onp.array([onp.iinfo(onp.int64).min, onp.iinfo(onp.int64).max, 0, -1, 1], dtype=onp.int64)
    yield onp.array([2 ** 53 + 1, 2 ** 53 + 3, 2 ** 53 - 1, 2 ** 53], dtype=onp.int64)
    yield onp.array([onp.iinfo(onp.int64).max, onp.iinfo(onp.int64).max - 1], dtype=onp.int64)
    yield onp.array([onp.finfo(f32).max, onp.finfo(f32).max], dtype=f32)
    yield onp.array([onp.finfo(f32).max] * 3, dtype=f32)  # odd count: numpy.ma.median's (h + h) / 2 overflows
    yield onp.array([onp.finfo(f32).max, onp.finfo(f32).max * onp.float32(0.75), 1.0, 2.0], dtype=f32)
    yield onp.array([onp.iinfo(onp.int32).min, onp.iinfo(onp.int32).max, 7], dtype=onp.int32)
    for n in (255, 256, 257, 2047, 2048, 2049, 8191, 8192, 8193):
        yield onp.random.default_rng(n).standard_normal(n)


def _check_edges(rb):
    for x in _edge_cases():
        X = rb.fromarray(x)
        for name in FUNCS:
            for q in (0.0, 0.5, 0.99, 1.0):
                if name.endswith("median") and q:
                    continue
                _check(rb, name, x, X, _q_for(name, q))
            if x.dtype.kind == "f":
                for m in ("lower", "midpoint", "hazen"):
                    if not name.endswith("median"):
                        _check(rb, name, x, X, _q_for(name, 0.5), method=m)
        x2 = onp.stack([x, x[::-1]])
        for name in FUNCS:
            _check(rb, name, x2, rb.fromarray(x2), _q_for(name, 0.5), axis=1)


def test_edge_values(q_engine):
    import ramba_b200 as rb

    _check_edges(rb)


def test_ranks_match_numpy_for_counts_past_the_exact_range_of_q():
    """The ranks of every method for counts around 2^24 (float32 q) and 2^53 (float64 q) equal NumPy's indexes computed
    with the count as a Python int, as NumPy computes them; a count array converted to float32 would round twice."""
    Q = sys.modules["ramba_b200.quantile"]
    for qdt, edges in ((onp.float32, (1 << 24,)), (onp.float64, (1 << 24, 1 << 53))):
        for m in METHODS:
            spec = Q._Spec("quantile", onp.array([0.5, 0.1, 0.3, 0.99, 1.0], dtype=qdt), m)
            for e in edges:
                counts = onp.array([e - 3, e - 1, e, e + 1, e + 3, e + 5, 7, 8], dtype=onp.int64)
                got = spec.ranks(counts, onp.dtype(qdt))
                for n, g in zip(counts, got):
                    idx = spec.indexes(int(n), onp.dtype(qdt))[0]
                    assert onp.array_equal(g, onp.clip(onp.where(idx < 0, n - 1, idx), 0, n - 1)), (qdt, m, int(n))
    # the array form alone, as it was, rounds n - 1 twice for float32 q at 2^24 + 3
    spec = Q._Spec("quantile", onp.array([0.5], dtype=onp.float32), "linear")
    n = (1 << 24) + 3
    twice = onp.floor((onp.float32(n) - onp.float32(1)) * onp.float32(0.5))
    assert twice != spec.indexes(n, onp.dtype(onp.float32))[0][0]


def test_float32_quantile_past_2_to_the_24(q_engine):
    """percentile / quantile / nanquantile of 2^24 + 3 float32 values (q float32, the pass form) equal NumPy's."""
    import ramba_b200 as rb

    x = _data(((1 << 24) + 3,), onp.float32, 14)
    X = rb.fromarray(x)
    _check(rb, "percentile", x, X, 50)
    _check(rb, "quantile", x, X, 0.5)
    _check(rb, "nanquantile", x, X, onp.float32(0.3))


def test_signed_zero_ties_compare_equal(q_engine):
    import ramba_b200 as rb

    x = onp.array([-0.0, 0.0, 0.0, -0.0])
    got = rb.median(rb.fromarray(x))
    assert got == onp.median(x) and got == 0.0


def _check_errors(rb):
    x = _data((4, 5), onp.float64, 8)
    X = rb.fromarray(x)
    for name in ("quantile", "nanquantile"):
        _check(rb, name, x, X, 1.5)
        _check(rb, name, x, X, [-0.1, 0.5])
    for name in ("percentile", "nanpercentile"):
        _check(rb, name, x, X, 101)
    _check(rb, "quantile", x, X, 0.5, method="nope")
    _check(rb, "quantile", x, X, onp.zeros((2, 2, 2)))
    _check(rb, "median", x, X, axis=2)
    for name in FUNCS:
        e = onp.zeros((0, 3))
        _check(rb, name, e, rb.fromarray(e), _q_for(name, 0.5))
        _check(rb, name, e, rb.fromarray(e), _q_for(name, 0.5), axis=0)
        _check(rb, name, e, rb.fromarray(e), _q_for(name, 0.5), axis=1)
    with pytest.raises(NotImplementedError):
        rb.median(X, axis=(0, 1))
    with pytest.raises(NotImplementedError):
        rb.quantile(X, 0.5, weights=X, method="inverted_cdf")
    with pytest.raises(NotImplementedError):
        rb.median(X, out=onp.empty(5))
    assert onp.median(X) == onp.median(x)  # NumPy dispatch
    assert onp.array_equal(onp.nanpercentile(X, [5, 50], axis=0).asarray(), onp.nanpercentile(x, [5, 50], axis=0))
    assert rb.median([1, 2, 3, 4]) == 2.5  # Python sequences go straight to NumPy


def test_errors_warnings_and_dispatch(q_engine):
    import ramba_b200 as rb

    _check_errors(rb)


# ---- the restatement ---------------------------------------------------------------------------------------------------------
def test_restatement_against_a_sort():
    r = onp.random.default_rng(9)
    for dt in (onp.float64, onp.float32, onp.int64, onp.int32):
        for n in (1, 2, 5, 300, 5000):
            x = (r.standard_normal(n) * 1e3).astype(dt)
            if dt in (onp.float64, onp.float32):
                x[r.random(n) < 0.1] = onp.nan
                x[r.random(n) < 0.1] = -0.0
                x[r.random(n) < 0.05] = onp.inf
            k = SV.keys_of(x)
            bits = x.dtype.itemsize * 8
            ranks = sorted(set([0, n - 1, n // 2, (n - 1) // 2] + list(r.integers(0, n, 5))))
            srt = onp.sort(k)
            for digit in (8, 11):
                assert onp.array_equal(SV.select(k, ranks, bits, digit), srt[ranks]), (dt, n, digit)
            assert onp.array_equal(SV.row_select(k, ranks, bits), srt[ranks])
            Q = sys.modules["ramba_b200.quantile"]

            assert onp.array_equal(Q.keys_of(x), k)
            back = Q.values_of(k, dt)
            assert onp.array_equal(back, x, equal_nan=True) and onp.array_equal(onp.signbit(back), onp.signbit(x) & ~onp.isnan(x)) or dt not in (onp.float64, onp.float32)


def test_checks_reject_wrong_restatements(q_engine, monkeypatch):
    """A key map that leaves a negative NaN uncanonicalised, and a choose step off by one rank, are both caught."""
    import ramba_b200 as rb

    x = onp.array([-onp.nan, 1.0, 2.0, 3.0, 0.5, 4.0])
    real = SV.keys_of

    def no_canon(v):
        v = onp.asarray(v)
        if v.dtype != onp.float64:
            return real(v)
        u = v.view(onp.uint64)
        sign = onp.uint64(1 << 63)
        return onp.where(u & sign, ~u, u | sign)

    monkeypatch.setattr(SV, "keys_of", no_canon)
    with pytest.raises(AssertionError):
        _check(rb, "nanmedian", x, rb.fromarray(x))
    monkeypatch.setattr(SV, "keys_of", real)
    _check(rb, "nanmedian", x, rb.fromarray(x))
    real_choose = SV.choose
    monkeypatch.setattr(SV, "choose", lambda st, p, bits, digit: real_choose(st, p, bits, digit, off_by_one=p == 0))
    y = _data((30000,), onp.float64, 10)  # the pass form
    with pytest.raises((AssertionError, RuntimeError)):
        _check(rb, "median", y, rb.fromarray(y))


# ---- the C-ABI -----------------------------------------------------------------------------------------------------------
def _view(shape, strides, eb=8, base=0x1000, bounds=None):
    from ramba_b200 import _cabi

    return _cabi.index_view(base, shape, strides, eb, bounds)


PLAN_CASES = [  # (shape, seg_len, targets, dtype code, segments)
    ([10 ** 9], 10 ** 9, 2, 0, 0), ([10 ** 9], 10 ** 9, 10, 1, 0), ([10 ** 9], 10 ** 9, 40, 0, 0), ([65536, 4096], 4096, 2, 0, 0),
    ([4096, 65536], 65536, 2, 0, 0), ([100, 12160], 12160, 2, 0, 0), ([100, 12161], 12161, 2, 0, 0), ([100, 24000], 24000, 3, 1, 0),
    ([7], 7, 1, 3, 0), ([5000], 5000, 2, 2, 1), ([3, 5000], 5000, 2, 0, 8), ([0], 1, 2, 0, 0),
]


def test_describe_select_plan_matches_the_restatement():
    from ramba_b200 import _cabi

    for shape, L, K, code, segs in PLAN_CASES:
        st = [int(onp.prod(shape[d + 1:])) for d in range(len(shape))]
        v = _view(shape, st, 4 if code in (1, 3) else 8)
        f = _cabi.group_plan_fields(_cabi.describe_select_plan(v, code, L, K, segs))
        exp = SV.plan(int(onp.prod(shape)), L, K, 32 if code in (1, 3) else 64, segs)
        for k, val in exp.items():
            assert f[k] == val, (shape, L, K, code, k, f[k], val)
        assert _cabi.select_scratch_bytes(v, code, L, K, segs) == exp["scratch_bytes"]
    assert SV.plan(65536 * 4096, 4096, 2, 64)["form"] == "row" and SV.plan(4096 * 65536, 65536, 2, 64)["form"] == "pass"


def test_no_select_row_switch(monkeypatch):
    from ramba_b200 import _cabi

    v = _view([64, 1000], [1000, 1])
    assert _cabi.group_plan_fields(_cabi.describe_select_plan(v, 0, 1000, 2))["form"] == "row"
    monkeypatch.setenv("RB200_NO_SELECT_ROW", "1")
    assert _cabi.group_plan_fields(_cabi.describe_select_plan(v, 0, 1000, 2))["form"] == "pass"


def test_malformed_arguments_are_rejected():
    from ramba_b200 import _cabi

    lib = _cabi.load()
    P = 0x1000

    def state(S=4, K=2):
        st = _cabi.SelectState()
        st.segments, st.targets = S, K
        for f in ("rank", "key", "slot", "slot_key", "n_slots", "counts", "nans", "matched", "cand", "cand_n"):
            setattr(st, f, P)
        st.cand_cap = 100
        return st

    def count(view=None, dtype=0, L=6, st=None, p=0, mode=0):
        v = view if view is not None else _view([4, 6], [6, 1])
        s = st if st is not None else state()
        return lib.rb200_select_count(C.byref(v), dtype, L, C.byref(s), p, mode, None), lib.rb200_last_error().decode()

    def rows(view=None, dtype=0, L=6, K=2, table=P, keys=P, nans=P):
        v = view if view is not None else _view([4, 6], [6, 1])
        return lib.rb200_select_rows(C.byref(v), dtype, L, K, table, 0, keys, nans, None), lib.rb200_last_error().decode()

    assert lib.rb200_select_count(C.byref(_view([4, 6], [6, 1])), 0, 6, None, 0, 0, None) != 0
    assert "null state" in lib.rb200_last_error().decode()
    assert "source dtype" in count(dtype=4, view=_view([4, 6], [6, 1], eb=1))[1]
    assert "elem_bytes does not match" in count(dtype=1)[1]
    assert "seg_len must be" in count(L=0)[1]
    assert "does not divide" in count(L=5)[1]
    assert "targets must be" in count(st=state(K=0))[1]
    assert "more segments than the array" in count(st=state(S=3))[1]
    assert "segments differ" in count(st=state(S=5))[1]
    assert "pass out of range" in count(p=8)[1]
    assert "bad mode" in count(mode=3)[1]
    assert "needs one segment" in count(p=1, mode=1)[1]
    one = _view([24], [1])
    assert "chosen prefix" in count(view=one, L=24, st=state(S=1), p=0, mode=1)[1]
    s = state(S=1)
    s.cand = None
    assert "candidate buffer" in count(view=one, L=24, st=s, p=1, mode=2)[1]
    s = state()
    s.counts = None
    assert "null state buffer" in count(st=s)[1]
    assert "null view base pointer" in count(view=_view([4, 6], [6, 1], base=0))[1]
    assert "outside its allocation" in count(view=_view([4, 6], [6, 1], bounds=(P, P + 20)))[1]
    assert "do not fit" in rows(view=_view([2, 50000], [50000, 1]), L=50000)[1]
    assert "null rank table" in rows(table=None)[1]
    assert lib.rb200_describe_select_plan(C.byref(_view([4, 6], [6, 1])), 0, 6, 0, 0) is None
    assert lib.rb200_select_scratch_bytes(C.byref(_view([4, 6], [6, 1])), 0, 7, 2, 0) == -1
    import torch

    if not torch.cuda.is_available():
        assert "no usable CUDA device" in count()[1]
        assert "no usable CUDA device" in rows()[1]


def test_header_and_exports_agree():
    from ramba_b200 import _cabi

    head = open(os.path.join(HERE, "..", "include", "ramba_b200.h")).read()
    for name in ("rb200_select_count", "rb200_select_choose", "rb200_select_rows", "rb200_select_scratch_bytes", "rb200_describe_select_plan"):
        assert name in _cabi.EXPORTS and re.search(r"\b%s\(" % name, head), name
    fields = re.search(r"typedef struct rb200_select_state \{(.*?)\} rb200_select_state;", head, re.S).group(1)
    names = re.findall(r"\b(\w+)(?:\[\w+\])?;", re.sub(r"/\*.*?\*/", "", fields, flags=re.S))
    assert names == [f for f, _ in _cabi.SelectState._fields_], (names, _cabi.SelectState._fields_)
    assert "#define RB200_ABI_VERSION 7" in head


def test_select_kernels_do_not_spill():
    """ptxas -v of rb200_select.cu (written by the build): no kernel spills to local memory."""
    log = os.path.join(HERE, "..", "ramba_b200", "csrc", "build", "rb200_select.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("library not built here")
    text = open(log).read()
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert spills and all(a == "0" and b == "0" for a, b in spills), spills
    assert text.count("Compiling entry function") == len(spills)


# ---- multi-rank over gloo ------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run_world(world, out, mode="oracle"):
    port = _free_port()
    procs = []
    for r in range(world):
        env = dict(os.environ)
        env.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r), "MASTER_ADDR": "127.0.0.1",
                    "MASTER_PORT": str(port), "OMP_NUM_THREADS": "1"})
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_quantile_worker.py"), out, mode], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=600)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, o))
    for rc, o in outs:
        assert rc == 0, o[-3000:]
    return dict(onp.load(out))


def _check_worlds(worlds):
    import _quantile_worker as QW

    npns = types.SimpleNamespace(fromarray=onp.asarray, median=onp.median, nanmedian=onp.nanmedian, quantile=onp.quantile,
                                 nanpercentile=onp.nanpercentile, percentile=onp.percentile, nanquantile=onp.nanquantile)
    x = QW.data()
    seen_cut = set()
    for name, call, ax, _ in QW.programs():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            e = onp.asarray(call(npns, x))
        for wd, res in worlds.items():
            g = res[name]
            if wd > 1 and ax is not None:
                seen_cut.add(bool(res[name + ".cut"]))
            assert g.dtype == e.dtype and g.shape == e.shape and onp.array_equal(g, e, equal_nan=True), (wd, name, g, e)
            assert onp.array_equal(g, worlds[1][name], equal_nan=True), (wd, name)
    for name, _, ax, K in QW.programs():
        for wd, res in worlds.items():
            n_coll, n_bytes = (int(v) for v in res[name + ".counters"])
            if wd == 1:
                assert n_coll == 0 and n_bytes == 0, (wd, name, n_coll, n_bytes)
            elif not bool(res[name + ".cut"]):
                # no exchange; a nan variant's 8-byte max all-reduce lets every rank warn together
                exp = (1, 8) if name.startswith("nan") else (0, 0)
                assert (n_coll, n_bytes) == exp, (wd, name, n_coll, n_bytes)
            else:
                GS, passes, digit, nan = QW.global_rows(name, x)
                # one sum all-reduce of the counts per pass, plus one of the nan counts after pass 0 (float data)
                assert n_coll == passes + nan, (wd, name, n_coll)
                assert n_bytes == passes * GS * K * (8 << digit) + nan * GS * 8, (wd, name, n_bytes)
    assert seen_cut == {True, False}, seen_cut  # both axis layouts ran


@pytest.fixture(scope="module")
def q_worlds(tmp_path_factory):
    d = tmp_path_factory.mktemp("quantile_worlds")
    return {w: _run_world(w, str(d / ("w%d.npz" % w))) for w in (1, 2, 3, 4, 8)}


@pytest.mark.timeout(1800)
def test_multirank_matches_one_rank_and_numpy(q_worlds):
    _check_worlds(q_worlds)


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_CODE = {onp.dtype(onp.float64): 0, onp.dtype(onp.float32): 1, onp.dtype(onp.int64): 2, onp.dtype(onp.int32): 3}


def _gpu_select_vs_vm(host, shape, strides, L, ranks, expect_form, force_pass=False, pad=16):
    """rb200_select_* over one view of device memory against a sort of the same keys, bit for bit; returns the plan."""
    import torch

    from ramba_b200 import _cabi

    dev = torch.device("cuda", 0)
    eb = host.dtype.itemsize
    code = _CODE[host.dtype]
    d_mem = torch.from_numpy(host.view(onp.uint8).copy()).to(dev)
    lo = sum(min(0, (s - 1) * st) for s, st in zip(shape, strides))
    base_off = (pad - lo) * eb
    view = _cabi.index_view(d_mem.data_ptr() + base_off, shape, strides, eb, (d_mem.data_ptr(), d_mem.data_ptr() + host.nbytes))
    h = onp.lib.stride_tricks.as_strided(host[pad:], shape, [s * eb for s in strides]).reshape(-1)
    keys = SV.keys_of(h)
    S, K = h.size // L, len(ranks)
    exp = onp.sort(keys.reshape(S, L), axis=1)[:, ranks]
    nanc = (keys.reshape(S, L) == SV.keys_of(onp.array([onp.nan], host.dtype))[0]).sum(axis=1) if host.dtype.kind == "f" else onp.zeros(S)
    plan = _cabi.group_plan_fields(_cabi.describe_select_plan(view, code, L, K))
    assert plan["form"] == expect_form, plan
    if plan["form"] == "row":
        table = torch.from_numpy(onp.array(ranks, onp.int64)).to(dev)
        out, nans = torch.zeros(S * K, dtype=torch.int64, device=dev), torch.zeros(S, dtype=torch.int64, device=dev)
        _cabi.select_rows(view, code, L, K, table.data_ptr(), False, out.data_ptr(), nans.data_ptr())
        got = out.cpu().numpy().view(onp.uint64).reshape(S, K)
        assert onp.array_equal(got, exp), (shape, host.dtype, plan)
        assert onp.array_equal(nans.cpu().numpy(), nanc)
        return plan, None
    digit, passes = plan["digit"], plan["passes"]
    t = lambda n, dt=torch.int64: torch.zeros(max(n, 1), dtype=dt, device=dev)  # noqa: E731
    st = _cabi.SelectState()
    st.segments, st.targets = S, K
    bufs = dict(rank=torch.from_numpy(onp.tile(onp.array(ranks, onp.int64), S)).to(dev), key=t(S * K), slot=t(S * K), slot_key=t(S * K),
                n_slots=t(S), counts=t((S * K) << digit), nans=t(S), matched=t(S), cand_n=t(1))
    for k, v in bufs.items():
        setattr(st, k, v.data_ptr())
    mode, modes, cand = _cabi.SELECT_READ, [], None
    for p in range(passes):
        _cabi.select_count(view, code, L, st, p, mode)
        modes.append(mode)
        if p == 0:
            assert onp.array_equal(bufs["nans"][:S].cpu().numpy(), nanc)
        _cabi.select_choose(view, code, L, st, p)
        if S == 1 and mode == _cabi.SELECT_READ and p + 2 < passes and not force_pass:
            m = int(bufs["matched"][0])
            if m <= max(h.size // 32, 65536):
                cand = t(m)
                st.cand, st.cand_cap = cand.data_ptr(), max(m, 1)
                mode = _cabi.SELECT_APPEND
        elif mode == _cabi.SELECT_APPEND:
            mode = _cabi.SELECT_CAND
    torch.cuda.synchronize()
    got = bufs["key"][:S * K].cpu().numpy().view(onp.uint64).reshape(S, K)
    assert onp.array_equal(got, exp), (shape, host.dtype, plan, modes)
    return plan, modes


def _host(dt, n, r, kind):
    if kind == "equal":
        return onp.full(n, 3, dtype=dt)
    x = (r.standard_normal(n) * 1e3).astype(dt)
    if dt in (onp.float64, onp.float32):
        x[r.random(n) < 0.05] = onp.nan
        x[r.random(n) < 0.05] = -0.0
    return x


@pytest.mark.gpu
def test_cuda_kernels_match_the_restatement(monkeypatch):
    r = onp.random.default_rng(0)
    seen = set()
    for dt in (onp.float64, onp.float32, onp.int64, onp.int32):
        for kind in ("spread", "equal"):
            # row form: rows of a 2-D view, contiguous and transposed
            host = _host(dt, 300 * 257 + 64, r, kind)
            _gpu_select_vs_vm(host, [300, 257], [257, 1], 257, [0, 128, 256, 100], "row")
            _gpu_select_vs_vm(host, [257, 300], [1, 257], 300, [0, 150, 149, 299], "row")
            # pass form, one segment: with candidate compaction on spread data
            host = _host(dt, 3_000_000 + 64, r, kind)
            plan, modes = _gpu_select_vs_vm(host, [3_000_000], [1], 3_000_000, [1_000_000, 2_000_000], "pass")
            seen.add(tuple(modes))
            _gpu_select_vs_vm(host, [1000, 3000], [3000, 1], 3000 * 1000, [7, 2_999_999], "pass")
            # pass form, many segments, strided (axis 0 of a 2-D array)
            host = _host(dt, 30000 * 40 + 64, r, kind)
            _gpu_select_vs_vm(host, [40, 30000], [1, 40], 30000, [0, 14999, 15000, 29999], "pass")
            # pass forced on a row-sized segment
            host = _host(dt, 64 * 1000 + 64, r, kind)
            monkeypatch.setenv("RB200_NO_SELECT_ROW", "1")
            _gpu_select_vs_vm(host, [64, 1000], [1000, 1], 1000, [0, 499, 500, 999], "pass", force_pass=True)
            monkeypatch.delenv("RB200_NO_SELECT_ROW")
            # many targets: several count-row groups per pass
            _gpu_select_vs_vm(host, [64 * 1000], [1], 64 * 1000, list(range(0, 64000, 400)), "pass")
    assert {(0, 0, 1, 2, 2, 2), (0, 0, 0, 0, 0, 0), (0, 0, 0)} <= seen, seen  # compaction on spread 64-bit keys only


@pytest.mark.gpu
def test_cuda_numpy_cases(gpu_engine):
    import ramba_b200 as rb

    _check_dtypes_and_ranks(rb)
    _check_methods_and_q(rb)
    _check_views(rb)
    _check_edges(rb)
    _check_errors(rb)


@pytest.mark.gpu
def test_cuda_benchmark_scale(gpu_engine):
    import ramba_b200 as rb

    r = onp.random.default_rng(12)
    x = r.standard_normal(20_000_000)
    X = rb.fromarray(x)
    _same(rb.median(X), onp.median(x), "median 2e7")
    _same(rb.percentile(X, [1, 25, 50, 75, 99]), onp.percentile(x, [1, 25, 50, 75, 99]), "percentile 2e7")
    xn = x.copy()
    xn[r.random(x.size) < 0.1] = onp.nan
    _same(rb.nanmedian(rb.fromarray(xn)), onp.nanmedian(xn), "nanmedian 2e7")
    y = r.standard_normal((4096, 1024))
    Y = rb.fromarray(y)
    _same(rb.median(Y, axis=1), onp.median(y, axis=1), "median axis 1")
    _same(rb.median(Y, axis=0), onp.median(y, axis=0), "median axis 0")
    f = x.astype(onp.float32)
    _same(rb.median(rb.fromarray(f)), onp.median(f), "median f32")


@pytest.mark.gpu
def test_cuda_float32_above_2_to_the_31():
    """2^31 + 5 float32 values, all but five equal: the target bucket holds more than 2^31 keys in every pass."""
    import torch

    from ramba_b200 import _cabi

    if torch.cuda.get_device_properties(0).total_memory < (40 << 30):
        pytest.skip("needs 40 GB")
    n = (1 << 31) + 5
    x = torch.full((n,), 1.5, dtype=torch.float32, device="cuda")
    x[:5] = torch.tensor([-1.0, 9.0, float("nan"), -0.0, 2.0])
    view = _cabi.index_view(x.data_ptr(), [n], [1], 4)
    plan = _cabi.group_plan_fields(_cabi.describe_select_plan(view, _cabi.F32, n, 2))
    assert plan["form"] == "pass"
    K, digit = 2, plan["digit"]
    t = lambda m, dt=torch.int64: torch.zeros(max(m, 1), dtype=dt, device="cuda")  # noqa: E731
    st = _cabi.SelectState()
    st.segments, st.targets = 1, K
    ranks = [n // 2, n - 2]
    bufs = dict(rank=torch.tensor(ranks, dtype=torch.int64, device="cuda"), key=t(K), slot=t(K), slot_key=t(K), n_slots=t(1),
                counts=t(K << digit), nans=t(1), matched=t(1), cand_n=t(1))
    for k, v in bufs.items():
        setattr(st, k, v.data_ptr())
    for p in range(plan["passes"]):
        _cabi.select_count(view, _cabi.F32, n, st, p, _cabi.SELECT_READ)
        _cabi.select_choose(view, _cabi.F32, n, st, p)
    torch.cuda.synchronize()
    got = bufs["key"].cpu().numpy().view(onp.uint64)
    exp = SV.keys_of(onp.array([1.5, 9.0], onp.float32))
    assert onp.array_equal(got, exp), (got, exp)
    assert int(bufs["nans"][0]) == 1 and int(bufs["matched"][0]) == n - 4
    del x
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_cuda_world2_over_nccl(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    one = _run_world(1, str(tmp_path / "w1.npz"), "cuda")
    two = _run_world(2, str(tmp_path / "w2.npz"), "cuda")
    _check_worlds({1: one, 2: two})
