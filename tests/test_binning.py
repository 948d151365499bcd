"""Binning: histogram, histogram_bin_edges, bincount, searchsorted and digitize.

CPU: the engine through the NumPy restatement of the kernels (_hist_vm) against NumPy with == on counts, indices and
edges, for every stored dtype, 0-d to 4-d, view kinds, lazy inputs and both DAG modes; edge values (every edge and one
ulp either side, bins=1, an empty range, infinities, NaN, int64 near 2^53, float32 edges), searchsorted ties, NaN and
signed zeros, digitize in both directions, and NumPy's errors; weighted sums against exact references within
gamma_{m-1+W-1} * sum|w| (each check shown to reject a wrong restatement); the restatement against a per-element brute
force; the plan, the argument checks and the exports of the C-ABI; no spills; gloo worlds 2, 3, 4 and 8 against world 1
and NumPy, with the transfer counters.
GPU: rb200_histogram / rb200_bin_search against the restatement bit for bit in every form and dtype and at chunk and
warp-step edges, a count above 2^32 in one bin; the NumPy cases through the CUDA library; world 2 over NCCL where two
GPUs exist."""
import ctypes as C
import fractions
import math
import os
import re
import socket
import subprocess
import sys
import types
import warnings

import numpy as onp
import pytest

import _hist_vm as HV
import _hist_worker as HW

HERE = os.path.dirname(os.path.abspath(__file__))
HV.extend_oracle_backend()  # (also for the oracle stand-in of the -m gpu tests under RB200_DRY_GPU_TESTS)
DTYPES = (onp.float64, onp.float32, onp.int64, onp.int32, onp.int16, onp.int8, onp.uint8, onp.uint16, onp.uint32)
SHAPES = [(), (7,), (5, 9), (3, 4, 5), (2, 3, 4, 5)]


@pytest.fixture
def hist_engine():
    import _oracle_backend
    from ramba_b200 import ramba
    from ramba_b200.runtime import RT

    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()
    _oracle_backend.install()
    yield
    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()


def _data(shape, dtype, seed):
    r = onp.random.default_rng(seed)
    dt = onp.dtype(dtype)
    if dt.kind == "f":
        return (r.standard_normal(shape) * 10).astype(dt)
    if dt == onp.bool_:
        return r.random(shape) < 0.5
    info = onp.iinfo(dt)
    return r.integers(max(info.min, -100), min(info.max, 100), size=shape, endpoint=True).astype(dt)


def _same(got, exp, what):
    from ramba_b200 import ndarray

    assert isinstance(got, ndarray), what
    g = got.asarray()
    exp = onp.asarray(exp)
    assert g.dtype == exp.dtype and g.shape == exp.shape, (what, g.dtype, exp.dtype, g.shape, exp.shape)
    assert onp.array_equal(g, exp, equal_nan=exp.dtype.kind == "f"), (what, g, exp)


def _check_hist(rb, x, X, **kw):
    h, e = rb.histogram(X, **kw)
    eh, ee = onp.histogram(x, **kw)
    _same(h, eh, ("histogram", x.dtype, x.shape, kw))
    _same(e, ee, ("edges", x.dtype, x.shape, kw))
    kw.pop("density", None)
    _same(rb.histogram_bin_edges(X, **kw), onp.histogram_bin_edges(x, **kw), ("histogram_bin_edges", kw))


BIN_CASES = [dict(), dict(bins=1), dict(bins=37), dict(bins=5, range=(-4, 6)), dict(bins=6, range=(-3.5, 7.25)),
             dict(bins=[-50, -3, 0, 0.5, 2, 60]), dict(bins=[-7, -2, 0, 1, 1, 9]), dict(bins=4, density=True)]


def _check_dtypes_and_ranks(rb):
    for dt in DTYPES:
        for i, shape in enumerate(SHAPES):
            x = _data(shape, dt, i)
            X = rb.fromarray(x) if shape else rb.array(x)
            if not shape:
                x = X.asarray()
            for kw in BIN_CASES:
                _check_hist(rb, x, X, **kw)
            f = x.reshape(-1)
            if shape and f.dtype.kind in "iu" and f.min() >= 0:
                _same(rb.bincount(rb.fromarray(f)), onp.bincount(f), ("bincount", dt))
            a = onp.sort(_data((23,), onp.float64, i + 7))
            if shape:
                for side in ("left", "right"):
                    _same(rb.searchsorted(a, X, side=side), onp.searchsorted(a, x, side=side).astype(onp.int64), ("searchsorted", dt, side))
                _same(rb.digitize(X, a[::3]), onp.digitize(x, a[::3]).astype(onp.int64), ("digitize", dt))
    b = onp.random.default_rng(1).random((6, 7)) < 0.4
    with pytest.warns(RuntimeWarning, match="Converting input from bool"):
        h, e = rb.histogram(rb.fromarray(b), bins=3, range=(0, 1))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        eh, ee = onp.histogram(b, bins=3, range=(0, 1))
    _same(h, eh, "bool histogram")
    _same(rb.bincount(rb.fromarray(b.reshape(-1))), onp.bincount(b.reshape(-1)), "bool bincount")


def test_every_dtype_and_rank(hist_engine):
    import ramba_b200 as rb

    _check_dtypes_and_ranks(rb)


VIEWS = [
    ("sliced", (9, 50), lambda x: x[1:8, 3:43]),
    ("stepped", (9, 90), lambda x: x[::2, ::3]),
    ("reversed", (5, 40), lambda x: x[::-1, ::-1]),
    ("transposed", (40, 7), lambda x: x.T),
    ("transposed3", (4, 6, 5), lambda x: x.transpose(2, 0, 1)),
    ("broadcast", (1, 40), lambda x: onp.broadcast_to(x, (4, 40)) if isinstance(x, onp.ndarray) else x.broadcast_to((4, 40))),
    ("lazy", (6, 40), lambda x: x * 2 - 1),
]


def _check_views(rb):
    for name, shape, view in VIEWS:
        for dt in (onp.float64, onp.float32, onp.int64, onp.int16):
            x = _data(shape, dt, 3)
            w = _data(shape, onp.float64, 4)
            hv, Xv = onp.asarray(view(x)), view(rb.fromarray(x))
            for kw in (dict(bins=9), dict(bins=[-30, -5, 0, 5, 30])):
                _check_hist(rb, hv, Xv, **kw)
            h, _ = rb.histogram(view(rb.fromarray(x)), bins=6, range=(-20, 20), weights=view(rb.fromarray(w)))
            _weighted_ok(onp.asarray(view(x)), onp.asarray(view(w)), 6, (-20, 20), h.asarray(), 1)
            a = onp.sort(_data((17,), dt, 5))
            _same(rb.searchsorted(a, view(rb.fromarray(x))), onp.searchsorted(a, hv).astype(onp.int64), ("searchsorted", name, dt))
    x = _data((12, 10), onp.float64, 4)  # a padded shard
    _check_hist(rb, x[2:9, 1:8], rb.fromarray(x, local_border=2)[2:9, 1:8], bins=7)
    lab = onp.arange(30) % 7
    L = rb.fromarray(lab)
    _same(rb.bincount(L[::-2]), onp.bincount(lab[::-2]), "reversed bincount")
    _same(rb.bincount(L * 2 + 1), onp.bincount(lab * 2 + 1), "lazy bincount")


def test_views_and_lazy_inputs(hist_engine):
    import ramba_b200 as rb

    _check_views(rb)


def _check_pending_and_no_dag(rb):
    x = _data((30, 20), onp.float64, 1)
    A = rb.fromarray(x)
    A[3:5] = 7.0  # a pending write to the input runs first
    y = x.copy()
    y[3:5] = 7.0
    _check_hist(rb, y, A, bins=11)
    _check_hist(rb, y * 3, A * 3, bins=[-40, 0, 7, 21, 22])
    h, _ = rb.histogram(A, bins=4)
    A[:, :] = 0.0  # written after the call: the result is concrete
    _same(h, onp.histogram(y, bins=4)[0], "written after")


def test_pending_inputs(hist_engine):
    import ramba_b200 as rb

    _check_pending_and_no_dag(rb)


def test_without_the_dag(hist_engine, monkeypatch):
    import ramba_b200 as rb
    from ramba_b200 import ramba

    monkeypatch.setattr(ramba, "NO_DAG", True)  # RAMBA_NO_DAG=1: statements go straight to the fuser
    _check_pending_and_no_dag(rb)
    _check_edge_values(rb)


# ---- edge values ---------------------------------------------------------------------------------------------------------
def _around(v):
    v = onp.asarray(v)
    return onp.concatenate([v, onp.nextafter(v, -onp.inf), onp.nextafter(v, onp.inf)])


def _check_edge_values(rb):
    for dt in (onp.float64, onp.float32):
        for bins, rng in ((10, (-1.0, 1.0)), (7, (0.1, 0.7)), (1, (-2.0, 3.0)), (33, (-1e-3, 5.0))):
            e = onp.histogram_bin_edges(onp.zeros(1, dt), bins, rng)
            x = _around(e.astype(dt)).astype(dt)
            _check_hist(rb, x, rb.fromarray(x), bins=bins, range=rng)
            x32 = onp.concatenate([x, onp.array([onp.inf, -onp.inf], dtype=dt)])
            _check_hist(rb, x32, rb.fromarray(x32), bins=bins, range=rng)
        edges = onp.array([-1.5, 0.0, 0.1, 0.1, 2.0], dtype=dt)
        x = onp.concatenate([_around(edges).astype(dt), onp.array([onp.nan, onp.inf, -onp.inf, -0.0], dtype=dt)])
        _check_hist(rb, x, rb.fromarray(x), bins=edges)
        _check_hist(rb, x, rb.fromarray(x), bins=list(edges.astype(onp.float64)))
        _check_hist(rb, x, rb.fromarray(x), bins=rb.fromarray(edges))
        y = onp.full(5, 3.25, dtype=dt)  # an empty range: NumPy widens it by 0.5
        _check_hist(rb, y, rb.fromarray(y), bins=4)
        _check_hist(rb, y, rb.fromarray(y), bins=4, range=(3.25, 3.25))
    big = onp.array([2 ** 53 - 2, 2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 53 + 2, 2 ** 53 + 3, 2 ** 60 + 1], dtype=onp.int64)
    for kw in (dict(bins=[float(2 ** 53 - 1), float(2 ** 53), float(2 ** 53 + 2), 2.0 ** 61]), dict(bins=[2 ** 53 - 1, 2 ** 53 + 1, 2 ** 53 + 3]),
               dict(bins=3), dict(bins=2, range=(2 ** 53 - 4, 2 ** 53 + 4)), dict(bins=3, range=(9007199254740991.0, 9007199254740995.0))):
        _check_hist(rb, big, rb.fromarray(big), **kw)
    for kw in (dict(bins=3), dict(bins=[0.0, 1.0]), dict(bins=4, range=(0, 1))):  # empty inputs
        _check_hist(rb, onp.zeros(0), rb.zeros((0,)), **kw)
    _same(rb.bincount(rb.zeros((0,), dtype=onp.int64)), onp.bincount(onp.zeros(0, dtype=onp.int64)), "empty bincount")
    _same(rb.bincount(rb.zeros((0,), dtype=onp.int64), minlength=3), onp.bincount(onp.zeros(0, dtype=onp.int64), minlength=3), "empty minlength")
    _same(rb.bincount(rb.fromarray(onp.array([3, 0, 3])), minlength=7), onp.bincount([3, 0, 3], minlength=7), "minlength")
    _same(rb.searchsorted([1.0, 2.0], rb.zeros((0, 3))), onp.zeros((0, 3), dtype=onp.int64), "empty search")


def test_edge_values(hist_engine):
    import ramba_b200 as rb

    _check_edge_values(rb)


def _check_search(rb):
    a = onp.array([-onp.inf, -2.0, -0.0, 0.0, 0.0, 1.0, 1.0, 1.0, 3.5, onp.inf, onp.nan, onp.nan])
    v = onp.array([[-onp.inf, -2.0, -1.0, -0.0, 0.0, 1.0, 2.0], [3.5, 4.0, onp.inf, onp.nan, 1.0, -3.0, 0.5]])
    for side in ("left", "right"):
        for A in (a, a.astype(onp.float32), rb.fromarray(a)):
            _same(rb.searchsorted(A, rb.fromarray(v), side=side), onp.searchsorted(onp.asarray(A) if not isinstance(A, rb.ndarray) else a, v, side=side).astype(onp.int64),
                  ("search", side))
        _same(rb.searchsorted(a, rb.fromarray(v.astype(onp.float32)), side=side), onp.searchsorted(a, v.astype(onp.float32), side=side).astype(onp.int64),
              ("search f32", side))
        ai = onp.array([2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 53 + 2], dtype=onp.int64)
        vf = onp.array([2.0 ** 53, 2.0 ** 53 + 2, 9007199254740993.0])
        _same(rb.searchsorted(ai, rb.fromarray(vf), side=side), onp.searchsorted(ai, vf, side=side).astype(onp.int64), ("int64 a, float64 v", side))
        vi = onp.array([2 ** 53 + 1, 2 ** 53 - 1, 5], dtype=onp.int64)
        _same(rb.searchsorted(ai, rb.fromarray(vi), side=side), onp.searchsorted(ai, vi, side=side).astype(onp.int64), ("int64 a, int64 v", side))
        _same(rb.searchsorted(ai.astype(onp.float64), rb.fromarray(vi), side=side), onp.searchsorted(ai.astype(onp.float64), vi, side=side).astype(onp.int64),
              ("float64 a, int64 v", side))
        s = rb.searchsorted(a, rb.array(onp.float64(1.0)), side=side)
        assert type(s) is onp.intp and s == onp.searchsorted(a, 1.0, side=side)
        assert rb.searchsorted(a, 1.0, side=side) == onp.searchsorted(a, 1.0, side=side)
    runs = onp.repeat(onp.arange(5), 7).astype(onp.int32)
    q = onp.arange(-1, 7).astype(onp.int16)
    for side in ("left", "right"):
        _same(rb.searchsorted(runs, rb.fromarray(q), side=side), onp.searchsorted(runs, q, side=side).astype(onp.int64), ("runs", side))
    _same(rb.fromarray(a).searchsorted(rb.fromarray(v), side="right"), onp.searchsorted(a, v, side="right").astype(onp.int64), "method")
    x = onp.array([-1.0, 0.0, 0.5, 1.0, 2.0, 2.5, 3.0, 4.0, onp.nan, -onp.inf])
    for bins in ([0.0, 1.0, 2.0, 3.0], [3.0, 2.0, 1.0, 0.0], [3.0, 3.0, 2.0, 0.0], [1.0, 1.0, 1.0], [2.0], [0, 1, 1, 3]):
        for right in (False, True):
            _same(rb.digitize(rb.fromarray(x), bins, right=right), onp.digitize(x, bins, right=right).astype(onp.int64), ("digitize", bins, right))
    _same(onp.digitize(rb.fromarray(x), onp.array([3.0, 1.0])), onp.digitize(x, [3.0, 1.0]).astype(onp.int64), "np.digitize")


def test_searchsorted_and_digitize(hist_engine):
    import ramba_b200 as rb

    _check_search(rb)


def _check_errors_and_dispatch(rb):
    x = _data((6, 7), onp.float64, 9)
    X = rb.fromarray(x)
    xn = x.copy()
    xn[2, 3] = onp.nan
    for call in (lambda m: m.histogram(xn), lambda m: m.histogram(xn, bins=3, range=(0, onp.inf)), lambda m: m.histogram(x, bins=[1, 0, 2]),
                 lambda m: m.histogram(x, bins=0), lambda m: m.histogram(x, bins=[[1, 2]]), lambda m: m.histogram(x, weights=onp.ones(3)),
                 lambda m: m.histogram(x, bins=3, range=(2, 1)), lambda m: m.bincount(onp.array([1, -1, 2])),
                 lambda m: m.bincount(onp.array([1, 2]), weights=onp.ones(3)), lambda m: m.bincount(onp.array([1, 2]), minlength=-1),
                 lambda m: m.bincount(onp.ones((2, 2), dtype=int)), lambda m: m.bincount(onp.array([1.0, 2.0])),
                 lambda m: m.digitize(x, [1.0, 0.0, 2.0]), lambda m: m.searchsorted([1.0, 2.0], x, side="middle"),
                 lambda m: m.histogram(x, bins=2.5)):
        with pytest.raises(Exception) as exp:
            call(onp)

        def conv(v):
            return rb.fromarray(v) if isinstance(v, onp.ndarray) and v.ndim else v

        ns = types.SimpleNamespace(histogram=lambda a, *k, **kw: rb.histogram(conv(a), *k, **{n: conv(w) for n, w in kw.items()}),
                                   bincount=lambda a, *k, **kw: rb.bincount(conv(a), *k, **{n: conv(w) for n, w in kw.items()}),
                                   digitize=lambda a, *k, **kw: rb.digitize(conv(a), *k, **kw),
                                   searchsorted=lambda a, v, **kw: rb.searchsorted(a, conv(v), **kw))
        with pytest.raises(exp.type):
            call(ns)
    for bins in ("auto", "fd"):
        with pytest.raises(NotImplementedError):
            rb.histogram(X, bins=bins)
    with pytest.raises(NotImplementedError):
        rb.searchsorted(onp.arange(3.0), X, sorter=onp.arange(3))
    with pytest.raises(NotImplementedError):
        rb.histogram(X[X > 0])
    with pytest.raises(NotImplementedError):
        rb.bincount(rb.fromarray(onp.arange(5))[rb.fromarray(onp.arange(5)) > 1])
    # NumPy's functions dispatch here
    h, e = onp.histogram(X, bins=5)
    _same(h, onp.histogram(x, bins=5)[0], "np.histogram")
    _same(onp.histogram_bin_edges(X, bins=5), onp.histogram_bin_edges(x, bins=5), "np.histogram_bin_edges")
    lab = onp.arange(20) % 6
    _same(onp.bincount(rb.fromarray(lab)), onp.bincount(lab), "np.bincount")
    _same(onp.searchsorted(onp.arange(5.0), X), onp.searchsorted(onp.arange(5.0), x).astype(onp.int64), "np.searchsorted")
    _same(onp.digitize(X, [0.0, 1.0]), onp.digitize(x, [0.0, 1.0]).astype(onp.int64), "np.digitize")


def test_errors_and_dispatch(hist_engine):
    import ramba_b200 as rb

    _check_errors_and_dispatch(rb)


# ---- weighted sums against exact references ------------------------------------------------------------------------------
def _gamma(k):
    u = fractions.Fraction(1, 2 ** 53)
    return k * u / (1 - k * u)


def _weighted_ok(x, w, bins, rng, got, world, out32=False, expect=None):
    """Every bin within gamma_{m-1+W-1} * sum|w| (+ one float32 rounding) of the exact sum of its weights."""
    x, w = onp.asarray(x).reshape(-1), onp.asarray(w, dtype=onp.float64).reshape(-1)
    idx = expect if expect is not None else None
    if idx is None:
        e = onp.histogram_bin_edges(x, bins, rng)
        idx = onp.array([onp.histogram(onp.array([v]), e)[0].argmax() if onp.histogram(onp.array([v]), e)[0].any() else -1 for v in x])
    for b in range(len(got)):
        mine = w[idx == b]
        m = mine.size
        g = float(got[b])
        if not onp.isfinite(mine).all():
            assert onp.isnan(g) if (onp.isnan(mine).any() or (onp.isposinf(mine).any() and onp.isneginf(mine).any())) else g == mine[~onp.isfinite(mine)][0], (b, g)
            continue
        exact = sum((fractions.Fraction(float(v)) for v in mine), fractions.Fraction(0))
        bound = _gamma(max(m - 1, 0) + world - 1) * sum(abs(fractions.Fraction(float(v))) for v in mine)
        err = abs(fractions.Fraction(g) - exact)
        if out32:
            bound += abs(exact) * fractions.Fraction(1, 2 ** 24) + bound
        assert err <= bound, (b, m, g, float(exact), float(err), float(bound))
        if m == 0 or all(v == 0 for v in mine):
            assert g == 0 and math.copysign(1, g) == 1, (b, g)


def _check_weighted(rb, world=1):
    r = onp.random.default_rng(3)
    lab = r.integers(0, 40, 5000)
    w = r.standard_normal(5000) * onp.exp(r.uniform(-20, 20, 5000))
    got = rb.bincount(rb.fromarray(lab), weights=rb.fromarray(w)).asarray()
    _weighted_ok(lab, w, None, None, got, world, expect=lab)
    wi = r.integers(-(2 ** 62), 2 ** 62, 5000)
    got = rb.bincount(rb.fromarray(lab), weights=rb.fromarray(wi)).asarray()
    _weighted_ok(lab, wi.astype(onp.float64), None, None, got, world, expect=lab)
    x = r.uniform(-1, 1, 3000)
    for wd in (onp.float64, onp.float32):
        ww = (r.standard_normal(3000) * 1e4).astype(wd)
        h, _ = rb.histogram(rb.fromarray(x), bins=12, range=(-1, 1), weights=rb.fromarray(ww))
        assert h.dtype == onp.dtype(wd)
        _weighted_ok(x, ww, 12, (-1, 1), h.asarray(), world, out32=wd == onp.float32)
        h, _ = rb.histogram(rb.fromarray(x), bins=[-1, -0.3, 0, 0.01, 1], weights=rb.fromarray(ww))
        _weighted_ok(x, ww, [-1, -0.3, 0, 0.01, 1], None, h.asarray(), world, out32=wd == onp.float32)
    # specials in one bin: NaN, +inf, inf - inf; -0.0 weights; an empty bin
    lab = onp.array([0, 0, 1, 1, 2, 2, 3, 3, 5])
    for sp in ([onp.nan, 1.0], [onp.inf, 2.0], [onp.inf, -onp.inf], [-0.0, -0.0]):
        wv = onp.array(sp + [1.0, 2.0, -0.0, -0.0, 4.0, 5.0, 6.0])
        got = rb.bincount(rb.fromarray(lab), weights=rb.fromarray(wv)).asarray()
        _weighted_ok(lab, wv, None, None, got, world, expect=lab)
        exp = onp.bincount(lab, wv)
        assert onp.array_equal(onp.signbit(got), onp.signbit(exp)) and onp.array_equal(onp.isnan(got), onp.isnan(exp)), (got, exp)


def test_weighted_sums_are_within_the_exact_bound(hist_engine):
    import ramba_b200 as rb

    _check_weighted(rb)


def test_weighted_checks_reject_a_wrong_restatement():
    """The bound checks above fail on deliberately wrong sums: a dropped element, a float32 accumulator, -0.0 kept."""
    r = onp.random.default_rng(4)
    lab = r.integers(0, 5, 400)
    w = r.standard_normal(400) * onp.exp(r.uniform(-10, 10, 400))
    right = onp.bincount(lab, w)
    dropped = onp.bincount(lab[1:], w[1:], minlength=5)
    f32 = onp.array([onp.float32(0)] * 5)
    for b, v in zip(lab, w):
        f32[b] = onp.float32(f32[b] + onp.float32(v))
    _weighted_ok(lab, w, None, None, right, 1, expect=lab)
    for wrong in (dropped, f32.astype(onp.float64)):
        with pytest.raises(AssertionError):
            _weighted_ok(lab, w, None, None, wrong, 1, expect=lab)
    with pytest.raises(AssertionError):
        _weighted_ok(onp.array([0]), onp.array([-0.0]), None, None, onp.array([-0.0]), 1, expect=onp.array([0]))


# ---- the restatement against a per-element brute force -------------------------------------------------------------------
def _numpy_fast_path(x, edges, first, last, n):
    """NumPy's equal-bins loop body on one element at a time (Python scalars of the dtypes it picks)."""
    from numpy.lib._histograms_impl import _unsigned_subtract

    out = []
    denom = _unsigned_subtract(last, first)
    for v in x:
        a = onp.array([v])
        if not ((a >= first) & (a <= last))[0]:
            out.append(-1)
            continue
        t = a.astype(edges.dtype)
        f = (_unsigned_subtract(t, first) / denom) * n
        i = int(f.astype(onp.intp)[0])
        i -= i == n
        i -= bool(t[0] < edges[i])
        i += bool(t[0] >= edges[i + 1] and i != n - 1)
        out.append(i)
    return onp.array(out)


def _brute_weighted(bins, wts, n, B, chunk, eb):
    """The library's fold order walked element by element."""
    E = 16 // eb
    ctas = -(-n // chunk) if n else 0
    out = [0.0] * B
    for c in range(ctas):
        rows = [[0.0] * B for _ in range(8)]
        p0, p1 = c * chunk, min((c + 1) * chunk, n)
        for b0 in range(p0, p1, 256 * E * 4):
            for wp in range(8):
                for k in range(4):
                    for u in range(E):
                        groups = {}
                        for lane in range(32):
                            p = b0 + wp * 32 * E * 4 + (k * 32 + lane) * E + u
                            if p < p1 and bins[p] >= 0:
                                groups.setdefault(bins[p], []).append(wts[p])
                        for b, vs in groups.items():
                            s = vs[0]
                            for v in vs[1:]:
                                s += v
                            rows[wp][b] += s
        for b in range(B):
            t = 0.0
            for wp in range(8):
                t += rows[wp][b]
            out[b] += t
    return onp.array(out)


def test_restatement_against_brute_force():
    r = onp.random.default_rng(0)
    for dt, rng in ((onp.float64, (-1.0, 1.0)), (onp.float32, (-1.0, 1.0)), (onp.float32, (0.1, 0.7)), (onp.int64, (-7, 12)), (onp.int64, (-7.5, 12.0))):
        for B in (1, 3, 10, 64):
            h = onp.zeros(0, dt)
            edges = onp.histogram_bin_edges(h, B, rng)
            from numpy.lib._histograms_impl import _get_outer_edges

            first, last = _get_outer_edges(h, rng)
            x = onp.concatenate([_around(edges.astype(dt)) if dt != onp.int64 else onp.arange(-9, 15), r.uniform(-1.5, 1.5, 50) * (10 if dt == onp.int64 else 1)]).astype(dt)
            from ramba_b200 import binning

            t = binning._table_for(onp.dtype(dt), edges, (first, last, B), types.SimpleNamespace(data_ptr=lambda: 0), edges.dtype)
            got = HV.bins_of(x, HV._table_dict(t), edges)
            assert onp.array_equal(got, _numpy_fast_path(x, edges, first, last, B)), (dt, rng, B)
    x = r.standard_normal(3 * 8192 + 77)
    bins = r.integers(-1, 6, x.size)
    bins[:2000] = 2  # a skewed stretch: whole warps in one bin
    w = r.standard_normal(x.size) * onp.exp(r.uniform(-30, 30, x.size))
    for eb in (8, 4):
        got = HV.weighted_sums(bins, w, x.size, 6, 8192, 4, eb)
        assert onp.array_equal(got, _brute_weighted(bins, w, x.size, 6, 8192, eb)), eb


# ---- the C-ABI -----------------------------------------------------------------------------------------------------------
def _view(shape, strides, eb=8, base=0x1000, bounds=None):
    from ramba_b200 import _cabi

    return _cabi.index_view(base, shape, strides, eb, bounds)


def _table(form, B, edge_dtype=0, edges=0x2000):
    from ramba_b200 import _cabi

    t = _cabi.BinTable()
    t.form, t.n_bins, t.edge_dtype, t.edges = form, B, edge_dtype, edges
    t.lo_dtype = t.hi_dtype = t.sub_dtype = t.div_dtype = 0
    t.denom = 1.0
    return t


PLAN_CASES = [  # (n, strides, weighted, form, B, edge dtype)
    (10 ** 9, 1, False, 0, 256, 0), (10 ** 9, 1, False, 0, 4096, 0), (10 ** 9, 1, False, 2, 10 ** 6, 0), (10 ** 9, 1, True, 2, 1000, 0),
    (10 ** 9, 1, True, 2, 4096, 0), (5000, 3, False, 1, 30000, 1), (8193, 1, True, 1, 12000, 0), (1, 1, False, 2, 1, 0), (0, 1, True, 0, 7, 1),
]


def test_describe_hist_plan_matches_the_restatement():
    from ramba_b200 import _cabi

    for n, st, weighted, form, B, edt in PLAN_CASES:
        f = _cabi.group_plan_fields(_cabi.describe_hist_plan(_view([n], [st]), weighted, _table(form, B, edt)))
        tb = 0 if form == 2 else (B + 1) * (4 if edt == 1 else 8)
        exp = HV.plan(n, B, weighted, tb)
        for k, v in exp.items():
            assert f[k] == v, (n, weighted, form, B, k, f[k], v)
        assert f["bins"] == B and f["warps"] == 8 and f["load"] == ("vector" if st == 1 else "strided")
        assert _cabi.histogram_scratch_bytes(_view([n], [st]), weighted, _table(form, B, edt)) == exp["scratch"]
    assert HV.plan(10 ** 9, 10 ** 6, False, 0)["form"] == "global" and HV.plan(10 ** 9, 4096, True, 0)["form"] == "slab"
    assert HV.plan(10 ** 9, 4096, True, 0)["passes"] == 3


def test_malformed_arguments_are_rejected():
    from ramba_b200 import _cabi

    lib = _cabi.load()
    P = 0x1000

    def hist(view=None, dtype=0, wview=None, wdt=0, table=None, out=P, bad=P):
        v = view if view is not None else _view([4, 6], [6, 1])
        t = table if table is not None else _table(0, 5)
        rc = lib.rb200_histogram(C.byref(v), dtype, C.byref(wview) if wview is not None else None, wdt, C.byref(t), out, bad, P, None)
        return rc, lib.rb200_last_error().decode()

    def search(view=None, dtype=0, tab=P, n=4, tdt=0, side=0, out=P):
        v = view if view is not None else _view([4, 6], [6, 1])
        return lib.rb200_bin_search(C.byref(v), dtype, tab, n, tdt, side, out, None), lib.rb200_last_error().decode()

    assert lib.rb200_histogram(C.byref(_view([3], [1])), 0, None, 0, None, P, P, P, None) != 0
    assert "null bin table" in lib.rb200_last_error().decode()
    assert "bad bin table form" in hist(table=_table(3, 5))[1]
    assert "n_bins" in hist(table=_table(0, 0))[1]
    assert "n_bins" in hist(table=_table(2, 1 << 31))[1]
    assert "uniform edges" in hist(table=_table(0, 5, edge_dtype=2))[1]
    assert "bad edge dtype" in hist(table=_table(1, 5, edge_dtype=3))[1]
    assert "null edges" in hist(table=_table(1, 5, edges=0))[1]
    t = _table(0, 5, edge_dtype=0)
    t.sub_dtype = 1
    assert "narrower" in hist(table=t)[1]
    assert "source dtype" in hist(dtype=4, view=_view([4, 6], [6, 1], eb=1))[1]
    assert "elem_bytes does not match" in hist(dtype=1)[1]
    assert "integer bins need an integer source" in hist(table=_table(2, 5))[1]
    assert "integer edges need" in hist(table=_table(1, 5, edge_dtype=2))[1]
    assert "differ in shape" in hist(wview=_view([4, 5], [5, 1]))[1]
    assert "weights dtype" in hist(wview=_view([4, 6], [6, 1], eb=1), wdt=5)[1]
    assert "null out" in hist(out=None)[1]
    assert "null bad" in hist(bad=None)[1]
    assert "null view base pointer" in hist(view=_view([4, 6], [6, 1], base=0))[1]
    assert "outside its allocation" in hist(view=_view([4, 6], [6, 1], bounds=(P, P + 20)))[1]
    assert "bad side" in search(side=2)[1]
    assert "null table" in search(tab=None)[1]
    assert "negative table length" in search(n=-1)[1]
    assert "table dtype" in search(tdt=3)[1]
    assert "integer table needs" in search(tdt=2)[1]
    assert "null out" in search(out=None)[1]
    assert lib.rb200_describe_hist_plan(C.byref(_view([4, 6], [6, 1])), 0, C.byref(_table(0, 0))) is None
    assert lib.rb200_histogram_scratch_bytes(C.byref(_view([4, 6], [6, 1])), 1, C.byref(_table(5, 3))) == -1
    import torch

    if not torch.cuda.is_available():
        assert "no usable CUDA device" in hist()[1]
        assert "no usable CUDA device" in search()[1]


def test_header_and_exports_agree():
    from ramba_b200 import _cabi

    head = open(os.path.join(HERE, "..", "include", "ramba_b200.h")).read()
    for name in ("rb200_histogram", "rb200_histogram_scratch_bytes", "rb200_describe_hist_plan", "rb200_bin_search"):
        assert name in _cabi.EXPORTS and re.search(r"\b%s\(" % name, head), name
    fields = re.search(r"typedef struct rb200_bin_table \{(.*?)\} rb200_bin_table;", head, re.S).group(1)
    names = re.findall(r"\b(\w+)(?:, (\w+))?;", re.sub(r"/\*.*?\*/", "", fields, flags=re.S))
    flat = [n for pair in names for n in pair if n]
    assert flat == [f for f, _ in _cabi.BinTable._fields_], (flat, _cabi.BinTable._fields_)
    assert "#define RB200_ABI_VERSION 7" in head


def test_hist_kernels_do_not_spill():
    """ptxas -v of rb200_hist.cu (written by the build): no kernel spills to local memory."""
    log = os.path.join(HERE, "..", "ramba_b200", "csrc", "build", "rb200_hist.ptxas.log")
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
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_hist_worker.py"), out, mode], env=env,
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


def _expected_programs():
    npns = types.SimpleNamespace(fromarray=onp.asarray, histogram=onp.histogram, bincount=onp.bincount, searchsorted=onp.searchsorted,
                                 digitize=onp.digitize)
    x, lab, w = HW.data()
    out = {}
    for name, call, _ in HW.programs():
        for i, e in enumerate(call(npns, x, lab, w)):
            out["%s.%d" % (name, i)] = onp.asarray(e)
    return out


# collectives at several ranks when the range or the length is found from the data: the min and the max all-reduce,
# then the sum all-reduce of the bins
FROM_DATA = 3


def _check_worlds(worlds):
    exp = _expected_programs()
    x, lab, w = HW.data()
    for wd, res in worlds.items():
        assert set(k for k in res if not k.endswith(".counters")) == set(exp), wd
        for k, e in exp.items():
            if k == "hist_weighted.0" or k == "bincount_w.0":
                assert res[k].dtype == e.dtype
                if k == "bincount_w.0":
                    _weighted_ok(lab, w, None, None, res[k], wd, expect=onp.concatenate([lab]))
                else:
                    _weighted_ok(lab * 0.5, w, 10, (0, 15), res[k], wd)
                continue
            assert res[k].dtype == e.dtype or (e.dtype == onp.intp and res[k].dtype == onp.int64), (wd, k)
            assert onp.array_equal(res[k], e), (wd, k, res[k], e)
            assert onp.array_equal(res[k], worlds[1][k]), (wd, k)
        for name, _, colls in HW.programs():
            n_coll, n_bytes = (int(v) for v in res[name + ".counters"])
            if wd == 1:
                assert n_coll == 0 and n_bytes == 0, (wd, name, n_coll)
            elif colls is not None:
                assert n_coll == colls, (wd, name, n_coll)
            else:
                assert n_coll == FROM_DATA, (wd, name, n_coll)


@pytest.fixture(scope="module")
def hist_worlds(tmp_path_factory):
    d = tmp_path_factory.mktemp("hist_worlds")
    return {w: _run_world(w, str(d / ("w%d.npz" % w))) for w in (1, 2, 3, 4, 8)}


@pytest.mark.timeout(1800)
def test_multirank_matches_one_rank_and_numpy(hist_worlds):
    _check_worlds(hist_worlds)


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_CODE = {onp.dtype(onp.float64): 0, onp.dtype(onp.float32): 1, onp.dtype(onp.int64): 2, onp.dtype(onp.int32): 3}


def _gpu_hist_vs_vm(host, shape, strides, table_kw, weights=None, pad=16, expect_form=None):
    """One view of device memory through rb200_histogram against the restatement on the same bytes, bit for bit."""
    import torch

    from ramba_b200 import _cabi, binning

    dev = torch.device("cuda", 0)
    eb = host.dtype.itemsize
    d_mem = torch.from_numpy(host.view(onp.uint8).copy()).to(dev)
    lo = sum(min(0, (s - 1) * st) for s, st in zip(shape, strides))
    base_off = (pad - lo) * eb
    view = _cabi.index_view(d_mem.data_ptr() + base_off, shape, strides, eb, (d_mem.data_ptr(), d_mem.data_ptr() + host.nbytes))
    h_view = _cabi.index_view(host.ctypes.data + base_off, shape, strides, eb)
    edges, uniform, form = table_kw["edges"], table_kw.get("uniform"), table_kw["form"]
    if form == _cabi.BINS_INTEGER:
        t = _cabi.BinTable()
        t.form, t.n_bins = form, table_kw["B"]
        d_edges = h_edges = None
    else:
        cmp = edges.dtype if uniform is not None else binning._edge_cmp(host.dtype, edges)
        d_edges = torch.from_numpy(onp.ascontiguousarray(edges, dtype=cmp)).to(dev)
        h_edges = onp.ascontiguousarray(edges, dtype=cmp)
        t = binning._table_for(host.dtype, edges, uniform, d_edges, cmp)
    B = int(t.n_bins)
    wview = h_wview = None
    if weights is not None:
        d_w = torch.from_numpy(weights).to(dev)
        wview = _cabi.index_view(d_w.data_ptr(), shape, [int(onp.prod(shape[d + 1:])) for d in range(len(shape))], weights.itemsize)
        h_wview = _cabi.index_view(weights.ctypes.data, shape, [int(onp.prod(shape[d + 1:])) for d in range(len(shape))], weights.itemsize)
    plan = _cabi.group_plan_fields(_cabi.describe_hist_plan(view, weights is not None, t))
    if expect_form:
        assert plan["form"] == expect_form, plan
    nsc = _cabi.histogram_scratch_bytes(view, weights is not None, t)
    scr = torch.empty(max(nsc, 1), dtype=torch.uint8, device=dev)
    out = torch.full((B,), 7, dtype=torch.float64 if weights is not None else torch.int64, device=dev)
    bad = torch.zeros(1, dtype=torch.int64, device=dev)
    wcode = _CODE[weights.dtype] if weights is not None else 0
    _cabi.histogram(view, _CODE[host.dtype], wview, wcode, t, out.data_ptr(), bad.data_ptr(), scr.data_ptr() if nsc else None)
    h_out = onp.full(B, 7, dtype=onp.float64 if weights is not None else onp.int64)
    h_bad = onp.zeros(1, dtype=onp.int64)
    if h_edges is not None:
        t.edges = h_edges.ctypes.data
    HV.histogram(h_view, _CODE[host.dtype], h_wview, wcode, t, h_out.ctypes.data, h_bad.ctypes.data)
    torch.cuda.synchronize()
    g = out.cpu().numpy()
    assert int(bad.cpu()[0]) == int(h_bad[0]), (int(bad.cpu()[0]), int(h_bad[0]))
    assert onp.array_equal(g.view(onp.int64), h_out.view(onp.int64)), (shape, strides, host.dtype, plan, g, h_out)
    return plan


def _uniform(dt, B, rng):
    from numpy.lib._histograms_impl import _get_outer_edges

    h = onp.zeros(0, dt)
    return {"form": 0, "edges": onp.histogram_bin_edges(h, B, rng), "uniform": _get_outer_edges(h, rng) + (B,)}


@pytest.mark.gpu
def test_cuda_histogram_matches_the_restatement():
    r = onp.random.default_rng(0)
    layouts = [([100003], [1]), ([37, 301], [301, 1]), ([37, 301], [1, 37]), ([40, 90], [-90, 3]), ([5, 6, 7, 8], [336, 56, 8, 1])]
    seen = set()
    for shape, strides in layouts:
        nmem = sum(abs((s - 1) * st) for s, st in zip(shape, strides)) + 1 + 32
        for dt in (onp.float64, onp.float32, onp.int64, onp.int32):
            f = dt in (onp.float64, onp.float32)
            host = (r.standard_normal(nmem) * 30).astype(dt) if f else r.integers(-5, 3000, nmem).astype(dt)
            n = int(onp.prod(shape))
            wts = [None, (r.standard_normal(n) * onp.exp(r.uniform(-20, 20, n))).reshape(shape), r.integers(-9, 9, n).astype(onp.int32).reshape(shape),
                   r.standard_normal(n).astype(onp.float32).reshape(shape)]
            cases = [_uniform(dt, 256, (-40, 40)), _uniform(dt, 4096, (-40.5, 40.0)), _uniform(dt, 30000, (-100, 3000)),
                     {"form": 1, "edges": onp.sort(r.standard_normal(300)) * 30}, {"form": 1, "edges": onp.sort(r.standard_normal(40000)) * 30}]
            if not f:
                cases += [{"form": 2, "B": 3001, "edges": None}, {"form": 2, "B": 30000, "edges": None}, {"form": 1, "edges": onp.arange(-5, 3000, 7)}]
            for tk in cases:
                for w in wts[:2] if tk.get("B", 0) != 30000 else wts[:1]:
                    plan = _gpu_hist_vs_vm(host, shape, strides, tk, weights=w)
                    seen.add((plan["form"], plan["table"]))
            _gpu_hist_vs_vm(host, shape, strides, cases[0], weights=wts[2])
            _gpu_hist_vs_vm(host, shape, strides, cases[0], weights=wts[3])
    assert {("shared", "shared"), ("global", "global"), ("slab", "global"), ("shared", "none"), ("global", "none")} <= seen, seen


@pytest.mark.gpu
def test_cuda_chunk_and_warp_step_edges():
    """Elements at CTA-chunk and warp-step edges, skewed stretches, the weighted fold bit for bit."""
    r = onp.random.default_rng(1)
    for dt, E in ((onp.float64, 2), (onp.float32, 4)):
        for n in (8191, 8192, 8193, 3 * 8192 + 1, 256 * E * 4 + 1, 32 * E * 4 - 1, 2 * 10 ** 6 + 3):
            host = r.uniform(-1, 1, n + 64).astype(dt)
            host[16 + 8192 - 40:16 + 8192 + 40] = 0.5  # one bin across a chunk edge
            w = r.standard_normal(n) * onp.exp(r.uniform(-25, 25, n))
            for tk in (_uniform(dt, 16, (-1, 1)), _uniform(dt, 2000, (-1, 1)), {"form": 1, "edges": onp.linspace(-1, 1, 17)}):
                _gpu_hist_vs_vm(host, [n], [1], tk)
                _gpu_hist_vs_vm(host, [n], [1], tk, weights=w)
    x = onp.zeros(8192 * 3 + 64, dtype=onp.int64)
    _gpu_hist_vs_vm(x, [8192 * 3], [1], {"form": 2, "B": 1, "edges": None}, expect_form="shared")
    _gpu_hist_vs_vm(x, [8192 * 3], [1], {"form": 2, "B": 1, "edges": None}, weights=onp.ones(8192 * 3), expect_form="shared")
    _gpu_hist_vs_vm(x, [8192 * 3], [1], {"form": 2, "B": 5000, "edges": None}, weights=onp.ones(8192 * 3), expect_form="slab")


@pytest.mark.gpu
def test_cuda_bin_search_matches_the_restatement():
    import torch

    from ramba_b200 import _cabi

    r = onp.random.default_rng(2)
    dev = torch.device("cuda", 0)
    for dt in (onp.float64, onp.float32, onp.int64, onp.int32):
        for m, tdt in ((0, onp.float64), (1, onp.float64), (1000, onp.float64), (30000, onp.float32), (20000, onp.int64)):
            if tdt == onp.int64 and dt in (onp.float64, onp.float32):
                continue
            tab = onp.sort((r.standard_normal(m) * 100).astype(tdt))
            if m > 10 and tdt != onp.int64:
                tab[-3:] = onp.nan
                tab[5:40] = tab[5]
            x = (r.standard_normal(70001) * 120).astype(dt)
            if dt in (onp.float64, onp.float32):
                x[::97] = onp.nan
                x[1::89] = -0.0
            if m:  # elements equal to table entries
                src = tab[::max(m // 100, 1)]
                src = src[~onp.isnan(src)] if src.dtype.kind == "f" else src
                x[2:2 + 50 * src.size:50] = src.astype(dt)
            d_x, d_t = torch.from_numpy(x).to(dev), torch.from_numpy(tab).to(dev) if m else torch.zeros(1, device=dev)
            for side in (0, 1):
                out = torch.full((x.size,), -5, dtype=torch.int64, device=dev)
                v = _cabi.index_view(d_x.data_ptr(), [x.size], [1], x.itemsize)
                _cabi.bin_search(v, _CODE[x.dtype], d_t.data_ptr() if m else None, m, _CODE[onp.dtype(tdt)], side, out.data_ptr())
                exp = onp.searchsorted(tab, x.astype(tdt), side="right" if side else "left")
                assert onp.array_equal(out.cpu().numpy(), exp), (dt, m, tdt, side)


@pytest.mark.gpu
def test_cuda_count_above_2_to_the_32():
    """2^32 + 3 int32 zeros in one bin, in the shared and the global form: 64-bit counts, positions and chunks."""
    import torch

    from ramba_b200 import _cabi

    if torch.cuda.get_device_properties(0).total_memory < (24 << 30):
        pytest.skip("needs 24 GB")
    n = (1 << 32) + 3
    x = torch.zeros(n, dtype=torch.int32, device="cuda")
    view = _cabi.index_view(x.data_ptr(), [n], [1], 4)
    bad = torch.zeros(1, dtype=torch.int64, device="cuda")
    for B, form in ((1, "shared"), (30000, "global")):
        t = _cabi.BinTable()
        t.form, t.n_bins = _cabi.BINS_INTEGER, B
        assert _cabi.group_plan_fields(_cabi.describe_hist_plan(view, False, t))["form"] == form
        out = torch.full((B,), 9, dtype=torch.int64, device="cuda")
        _cabi.histogram(view, _cabi.I32, None, 0, t, out.data_ptr(), bad.data_ptr(), None)
        torch.cuda.synchronize()
        assert int(out[0]) == n and int(out[1:].sum()) == 0 and int(bad[0]) == 0, (B, int(out[0]))
    del x
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_cuda_numpy_cases(gpu_engine):
    import ramba_b200 as rb

    _check_dtypes_and_ranks(rb)
    _check_views(rb)
    _check_pending_and_no_dag(rb)
    _check_edge_values(rb)
    _check_search(rb)
    _check_errors_and_dispatch(rb)
    _check_weighted(rb)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_cuda_world2_over_nccl(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    one = _run_world(1, str(tmp_path / "w1.npz"), "cuda")
    two = _run_world(2, str(tmp_path / "w2.npz"), "cuda")
    _check_worlds({1: one, 2: two})
