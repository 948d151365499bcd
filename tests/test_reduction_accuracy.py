"""Accumulation accuracy of every reduction and scan, held to exact host references.

Every float reduction and scan accumulates in float64 and rounds once to the result dtype (DESIGN §6).  Integer-valued
data cannot tell that apart from a float32 accumulator, so the data here are chosen where the accumulator's width shows:

  * family A: x = m * 2^e with full-width mantissas (24 bits for float32, up to 29 for float64) and e in [E0, E0 + K],
    K chosen so that n * 2^(mbits + K) < 2^53.  Every partial sum, in any order, is then exact in float64, and almost
    none is exact in float32.  The exact total is int64 arithmetic on x * 2^-E0; a float32 result must be that integer
    rounded once to float32 (then scaled), bit for bit, and a float64 result the integer itself.  Any narrowing to
    float32 on the way, any dropped or doubled element or partial and any wrong combine shows in the bits.
  * family B: inexact float64 (several decades, cancelling pairs).  The reference is exact (math.fsum, Python-int
    prefix sums); the result must lie within 1/2 ulp(exact) + gamma_d * sum|x|, gamma_d = d u / (1 - d u), u = 2^-53, d
    the longest chain of additions from an element to the result.
  * specials, bit for bit against NumPy: NaN and infinities in sums, float32 overflow, the sign of zero, and min / max
    with one NaN at every position class (a NaN anywhere gives NaN).

The CPU tests run the engine on the oracle backend (the NumPy restatement of the kernels), over gloo worlds of 1 to 8
ranks, and show that each check fails on a deliberately wrong host restatement.  The GPU tests run the same checks on the
kernels, each case asserting through rb200_describe_plan the kernel form it is meant to reach, in one process per set of
kernel switches (RB200_NO_*, read once per process)."""
import json
import math
import os
import socket
import subprocess
import sys
from fractions import Fraction

import numpy as onp
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
U64 = 2.0 ** -53


# ---- family A ---------------------------------------------------------------------------------------------------------
def family_a(shape, dtype, seed, mbits=None, e0=-20):
    """(x, ints, E0): x = ints * 2^E0 exactly, ints int64 with full-width mantissas, sum |ints| < 2^53."""
    n = int(onp.prod(shape))
    if mbits is None:
        mbits = 24 if dtype == onp.float32 else min(29, 51 - max(1, n - 1).bit_length())
    k = 52 - mbits - max(1, n - 1).bit_length()
    assert k >= 0 and (dtype != onp.float32 or mbits <= 24), (shape, dtype, mbits)
    r = onp.random.default_rng(seed)
    lo = 1 << (mbits - 1)
    m = r.integers(lo, 2 * lo, size=n, dtype=onp.int64) * r.choice([-1, 1], size=n)
    ints = (m << r.integers(0, k + 1, size=n)).reshape(shape)
    assert int(onp.abs(ints).sum()) < 2 ** 53
    x = onp.ldexp(ints.astype(onp.float64), e0).astype(dtype)
    assert onp.array_equal(onp.ldexp(x.astype(onp.float64), -e0), ints.astype(onp.float64))
    return x, ints, e0


def exact_ints(y):
    """(ints, E) with y = ints * 2^E exactly for any finite float array y whose exact sum fits 53 bits in every order."""
    y = onp.asarray(y)
    f = y.astype(onp.float64)
    nz = f[f != 0]
    if nz.size == 0:
        return onp.zeros(y.shape, dtype=onp.int64), 0
    mant, ex = onp.frexp(nz)
    m = onp.abs(onp.ldexp(mant, 53).astype(onp.int64))
    e = int((ex - 53 + onp.log2(m & -m).astype(onp.int64)).min())  # the lowest set bit of any element
    ints = onp.ldexp(f, -e).astype(onp.int64)
    assert int(onp.abs(ints).sum()) < 2 ** 53, "data are not family A"
    return ints, e


def round_to(ints, e, dtype):
    """ints * 2^e rounded once to dtype (the float64 conversion is exact: |ints| < 2^53)."""
    return onp.ldexp(onp.asarray(ints).astype(onp.float64), e).astype(dtype)


def want_sum(y, dtype, axis=None):
    ints, e = exact_ints(y)
    return round_to(ints.sum(axis=axis), e, dtype)


def want_cumsum(y, dtype, axis):
    ints, e = exact_ints(y)
    return round_to(onp.cumsum(ints, axis=axis), e, dtype)


def want_mean(y, dtype, axis=None):
    """The engine's formula on the exact sum: s / n globally (NumPy scalar arithmetic), s * (1.0 / n) along an axis (the
    loop body computes a float32 s times a Python float in float64 and stores float32), within 1 ulp of S / n."""
    s = want_sum(y, dtype, axis)
    n = y.size if axis is None else y.shape[axis]
    m = dtype(s / n) if axis is None else (s.astype(onp.float64) * (1.0 / n)).astype(dtype)
    ints, e = exact_ints(y)
    few = onp.atleast_1d(ints.sum(axis=axis))[:64]
    exact = onp.array([float(Fraction(int(v), n) * Fraction(2) ** e) for v in few]).astype(dtype)
    assert (onp.abs(onp.atleast_1d(m)[:64].astype(onp.float64) - exact) <= onp.spacing(onp.abs(exact))).all()
    return m


def want_prod(y, dtype):
    """Product of data +-2^k * {1, 3} (at most 33 threes: exact in float64), rounded once to dtype."""
    p = Fraction(1)
    for v in y.reshape(-1).astype(onp.float64):
        p *= Fraction(float(v))
    return dtype(float(p))


def prod_data(n, dtype, seed):
    r = onp.random.default_rng(seed)
    x = onp.ldexp(onp.where(r.random(n) < 0.5, 1.0, -1.0), r.integers(-1, 2, size=n))
    x[r.choice(n, size=min(n, 33), replace=False)] *= 3.0
    return x.astype(dtype)


def same_bits(got, want):
    """Number of elements whose bits differ (any NaN matches any NaN)."""
    got, want = onp.ascontiguousarray(onp.atleast_1d(got)), onp.ascontiguousarray(onp.atleast_1d(want))
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    bad = (got.view(onp.uint8).reshape(got.shape + (-1,)) != want.view(onp.uint8).reshape(want.shape + (-1,))).any(axis=-1)
    if got.dtype.kind == "f":
        bad &= ~(onp.isnan(got) & onp.isnan(want))
    return int(bad.sum())


def assert_bits(got, want, what=""):
    nbad = same_bits(got, want)
    if nbad:
        got, want = onp.asarray(got).reshape(-1), onp.asarray(want).reshape(-1)
        raise AssertionError("%s: %d of %d differ, e.g. got %r want %r" % (what, nbad, got.size, got[:4], want[:4]))


# ---- family B ---------------------------------------------------------------------------------------------------------
def family_b(n, seed, kind):
    r = onp.random.default_rng(seed)
    if kind == "decades":
        return r.choice([-1.0, 1.0], size=n) * 10.0 ** r.uniform(-6, 6, size=n)
    x = r.uniform(-1, 1, size=n // 2) * 10.0 ** r.integers(0, 8, size=n // 2)  # x, -x pairs plus small terms
    y = onp.concatenate([x, -x[r.permutation(x.size)]])
    y[r.choice(y.size, size=max(1, n // 100), replace=False)] = r.uniform(-1e-3, 1e-3, size=max(1, n // 100))
    return onp.concatenate([y, r.uniform(-1, 1, size=n - y.size)])


def gamma(d):
    return d * U64 / (1 - d * U64)


def sum_error_ratio(got, x, d):
    """|got - exact| / (1/2 ulp(exact) + gamma_d sum|x|) for a float64 sum of x."""
    x = [float(v) for v in onp.asarray(x).reshape(-1)]
    s1 = math.fsum(x)
    s2 = math.fsum(x + [-s1])  # the residual of the rounded total: s1 + s2 + s3 is the exact sum to 2^-150 relative
    exact = Fraction(s1) + Fraction(s2) + Fraction(math.fsum(x + [-s1, -s2]))
    bound = Fraction(onp.spacing(abs(float(exact)))) / 2 + Fraction(gamma(d)) * Fraction(math.fsum(onp.abs(x)))
    return float(abs(Fraction(float(got)) - exact) / bound)


def prod_error_ratio(got, x, d):
    """|got - exact| / (1/2 ulp(exact) + gamma_d |exact|) for a float64 product of d + 1 positive terms (every
    multiplication rounds once, in any order), the exact product from mpmath at 200 bits."""
    import mpmath

    with mpmath.workprec(200):
        exact = mpmath.fprod([mpmath.mpf(float(v)) for v in x])
        bound = mpmath.mpf(float(onp.spacing(float(exact)))) / 2 + mpmath.mpf(gamma(d)) * abs(exact)
        return float(abs(mpmath.mpf(float(got)) - exact) / bound)


def cumsum_error_ratio(got, x, d):
    """max over i of |got_i - exact prefix_i| / (1/2 ulp + gamma_d sum_{j<=i} |x_j|): Python-int prefixes on 2^-k."""
    ints, e = _scaled(x)
    ex = onp.array([Fraction(v) for v in _pyint_cumsum(ints)], dtype=object)
    ab = _pyint_cumsum([abs(v) for v in ints])
    worst = 0.0
    step = max(1, len(x) // 4096)
    for i in list(range(0, len(x), step)) + [len(x) - 1]:
        exact = ex[i] * Fraction(2) ** e
        bound = Fraction(onp.spacing(abs(float(exact)))) / 2 + Fraction(gamma(d)) * Fraction(ab[i]) * Fraction(2) ** e
        worst = max(worst, float(abs(Fraction(float(got[i])) - exact) / bound))
    return worst


def _scaled(x):
    _, ex = onp.frexp(x[x != 0])
    e = int(ex.min()) - 53
    return [int(v) for v in onp.ldexp(x, -e).astype(object)], e


def _pyint_cumsum(v):
    out, s = [], 0
    for a in v:
        s += int(a)
        out.append(s)
    return out


# ---- kernel forms: the longest chain of additions from an element to the result ---------------------------------------
def chain_global(n):
    """Any global or axis form: work is handed out in groups of 16 consecutive elements, and at least one CTA of 256
    threads folds the n elements, so one thread folds at most 16 * ceil(n / 4096) elements serially (its groups and its
    in-thread tree together), then warp (5), CTA (3), the fold of at most 2^17 CTA or split partials (17) and the final
    red[0] step (1)."""
    return 16 * -(-n // 4096) + 5 + 3 + 17 + 1


def chain_any(m):
    """Any order of summing m terms (the grouped kernels' chunks, splits and fold): at most m - 1 additions."""
    return max(1, m - 1)


def chain_scan(n):
    """Scans: an inclusive prefix is at most one addition per preceding element plus the carry of the earlier tiles
    or ranks (look-back: tile aggregate + prefix; columns: serial)."""
    return n + 2


# ---- deliberately wrong host restatements (each check must fail on them) ----------------------------------------------
CTA = 256


def restated_sum(x, acc=onp.float64, drop=False, double_partial=False, round_partial=False):
    """Column sums of a 2-D x in the shape of the kernels: one serial partial per CTA of CTA rows, then the fold of the
    partials.  acc: accumulator dtype; drop: lose the last row; double_partial: fold the second CTA partial twice;
    round_partial: round each CTA partial to float32 before the fold."""
    x = onp.asarray(x)
    if drop:
        x = x[:-1]
    parts = []
    for i in range(0, x.shape[0], CTA):
        s = onp.zeros(x.shape[1:], dtype=acc)
        for row in x[i:i + CTA].astype(acc):
            s = (s + row).astype(acc)
        parts.append(s.astype(onp.float32).astype(acc) if round_partial else s)
    if double_partial and len(parts) > 1:
        parts.append(parts[1])
    tot = onp.zeros(x.shape[1:], dtype=acc)
    for p in parts:
        tot = (tot + p).astype(acc)
    return tot


def restated_min(x, combine):
    """Tree min with the given combine(a, b), from the identity +inf (red[0] = red[0] (op) acc)."""
    v = [float(t) for t in onp.asarray(x).reshape(-1)]
    while len(v) > 1:
        v = [combine(v[i], v[i + 1]) if i + 1 < len(v) else v[i] for i in range(0, len(v), 2)]
    return combine(math.inf, v[0])


def old_min(a, b):
    return b if b < a else a


def nan_min(a, b):
    return b if (b < a or b != b) else a


def test_family_a_is_exact_in_float64_and_not_in_float32():
    x, ints, e0 = family_a((100003,), onp.float32, 1)
    assert int(onp.count_nonzero(onp.cumsum(x.astype(onp.float32), dtype=onp.float32) != round_to(onp.cumsum(ints), e0, onp.float32))) > 90000
    assert onp.cumsum(x.astype(onp.float64))[-1] == onp.ldexp(float(ints.sum()), e0)
    y, yi, _ = family_a((1 << 20,), onp.float64, 2)
    assert onp.abs(yi).max() >= 2 ** 28 and onp.count_nonzero(y.astype(onp.float32).astype(onp.float64) != y) > 1000


def test_each_check_fails_on_a_wrong_restatement():
    wrongs = (dict(acc=onp.float32), dict(drop=True), dict(double_partial=True), dict(round_partial=True))
    for dt in (onp.float32, onp.float64):
        x, _, _ = family_a((2053, 64), dt, 3)
        want = want_sum(x, dt, 0)
        assert_bits(restated_sum(x).astype(dt), want)
        for wrong in wrongs:
            assert same_bits(restated_sum(x, **wrong).astype(dt), want) > 0, (dt, wrong)
        assert same_bits(onp.cumsum(x, axis=0, dtype=onp.float32).astype(dt), want_cumsum(x, dt, 0)) > x.size // 2
    # family B: the bound holds for the float64 restatement and fails for a float32 accumulator
    xb = family_b(50003, 5, "decades")[:, None]
    assert sum_error_ratio(restated_sum(xb)[0], xb, chain_global(xb.size)) <= 1.0
    assert sum_error_ratio(restated_sum(xb, acc=onp.float32)[0], xb, chain_global(xb.size)) > 1.0
    # groupby var: the two-pass form stays inside var_bound, the one-pass E[x^2] - E[x]^2 does not
    xv = 1e8 + onp.random.default_rng(6).standard_normal(20000)
    exact, bound = var_bound(xv, chain_any(xv.size))
    c = xv.sum() / xv.size
    assert abs(Fraction(float(((xv - c) ** 2).sum() / xv.size)) - exact) <= bound
    assert abs(Fraction(float(var_one_pass(xv))) - exact) > bound
    # min / max: the old combine loses a NaN at some position, the NaN-propagating one never does
    for n in (7, 16, 33):
        lost = 0
        for p in range(n):
            v = onp.arange(n, dtype=onp.float64)
            v[p] = onp.nan
            assert math.isnan(restated_min(v, nan_min))
            lost += not math.isnan(restated_min(v, old_min))
        assert lost > 0


# ---- engine cases, shared by the oracle and the GPU tests ---------------------------------------------------------------
def _cases(size):
    """[(name, form, build(rb) -> {label: (got, want, kind)})]: kind "bits" (bit for bit) or a family B bound.  form: the
    plan (rb200_describe_plan, rb200_describe_group_plan, the scan form, the fold of split partials) the case must reach:
    a prefix, a predicate, or a tuple of them that must all be met."""
    big = size == "big"
    n1 = (1 << 26) + 12345 if big else 100003        # grid-stride loops with several iterations per thread, ragged tail
    nscan = 2400 * 2048 + 4099 if big else 70001      # more than 2400 look-back tiles
    rows = (1 << 20) + 7 if big else 4099             # split axis reductions
    cases = []

    def add(name, form, fn):
        cases.append((name, form, fn))

    for dt in (onp.float32, onp.float64):
        tag = "f32" if dt == onp.float32 else "f64"
        x, _, _ = family_a((n1,), dt, 10)
        add("sum_%s" % tag, "kernel=stream mode=elementwise", lambda rb, x=x, dt=dt: {"sum": (rb.fromarray(x).sum(), want_sum(x, dt), "bits")})
        add("mean_%s" % tag, "kernel=stream mode=elementwise", lambda rb, x=x, dt=dt: {"mean": (rb.fromarray(x).mean(), want_mean(x, dt), "bits")})
        add("map_sum_%s" % tag, "kernel=mapred mode=global",
            lambda rb, x=x, dt=dt: {"sum": ((rb.fromarray(x) * -2.0).sum(), want_sum(x.astype(dt) * dt(-2.0), dt), "bits")})
        y, _, _ = family_a((n1,), dt, 11, mbits=20 if dt == onp.float32 else None)
        z, _, _ = family_a((n1,), dt, 12, mbits=20 if dt == onp.float32 else None)
        add("two_source_sum_%s" % tag, "kernel=stream_terms",
            lambda rb, y=y, z=z, dt=dt: {"sum": ((rb.fromarray(y) - rb.fromarray(z)).sum(), want_sum((y - z).astype(dt), dt), "bits")})
        add("strided_sum_%s" % tag, "kernel=stream mode=elementwise", lambda rb, x=x, dt=dt: {"sum": (rb.fromarray(x)[::3].sum(), want_sum(x[::3], dt), "bits")})
        add("reversed_sum_%s" % tag, "kernel=stream mode=elementwise", lambda rb, x=x, dt=dt: {"sum": (rb.fromarray(x)[::-1].sum(), want_sum(x[::-1], dt), "bits")})
        add("sin_sum_%s" % tag, "kernel=general_interpreter",  # outside the streaming vocabulary: the interpreter's reduction
            lambda rb, x=x, dt=dt: {"sum": ((rb.fromarray(x) + 0.0 * rb.sin(rb.fromarray(x))).sum(), want_sum(x, dt), "bits")})
        s, _, _ = family_a((nscan,), dt, 13)
        add("cumsum_%s" % tag, lambda p, big=big: p.startswith("kernel=scan form=lookback") and (not big or int(p.split("tiles=")[1]) > 2400), lambda rb, s=s, dt=dt: {"cumsum": (rb.cumsum(rb.fromarray(s)), want_cumsum(s, dt, 0), "bits")})
        for shape in ((rows, 37), (37, rows)):
            m, _, _ = family_a(shape, dt, 14 + shape[0] % 7)
            for ax in (0, 1):
                add("axis%d_sum_%s_%dx%d" % (ax, tag, shape[0], shape[1]), AXIS_SPLIT,
                    lambda rb, m=m, ax=ax, dt=dt: {"sum": (rb.fromarray(m).sum(axis=ax), want_sum(m, dt, ax), "bits"),
                                                   "mean": (rb.fromarray(m).mean(axis=ax), want_mean(m, dt, ax), "bits")})
                add("axis%d_cumsum_%s_%dx%d" % (ax, tag, shape[0], shape[1]), "kernel=scan form=lookback" if ax == 1 else "kernel=scan form=columns",
                    lambda rb, m=m, ax=ax, dt=dt: {"cumsum": (rb.cumsum(rb.fromarray(m), axis=ax), want_cumsum(m, dt, ax), "bits")})
            add("transposed_sum_%s_%dx%d" % (tag, shape[0], shape[1]), AXIS_SPLIT,
                lambda rb, m=m, dt=dt: {"sum": (rb.fromarray(m).T.sum(axis=0), want_sum(m.T, dt, 0), "bits")})
        cx, _, _ = family_a((4097 if big else 3001, 4096), dt, 24, mbits=20 if dt == onp.float32 else None)
        cy, _, _ = family_a(cx.shape, dt, 25, mbits=20 if dt == onp.float32 else None)
        cv = cy[0].copy()
        for cname, cform, make, ref in (
                ("plain", "kernel=stream mode=columns", lambda rb, X, Y, v: X, lambda x, y, v: x),
                ("scaled", "kernel=mapred mode=columns", lambda rb, X, Y, v: X * 2.0, lambda x, y, v: x * x.dtype.type(2.0)),
                ("broadcast", "kernel=mapred mode=columns", lambda rb, X, Y, v: X + v, lambda x, y, v: x + v),
                ("two_source", "kernel=stream_terms mode=columns", lambda rb, X, Y, v: X - Y, lambda x, y, v: x - y),
                ("interpreter", "kernel=general_interpreter form=axis_as_1d", lambda rb, X, Y, v: X + 0.0 * rb.sin(X), lambda x, y, v: x)):
            add("columns_%s_%s" % (cname, tag), cform, lambda rb, make=make, ref=ref, dt=dt, cx=cx, cy=cy, cv=cv: {
                "sum": (make(rb, rb.fromarray(cx), rb.fromarray(cy), rb.fromarray(cv)).sum(axis=0), want_sum(ref(cx, cy, cv).astype(dt), dt, 0), "bits")})
        p = prod_data(4099, dt, 15)
        add("prod_%s" % tag, "kernel=stream mode=elementwise", lambda rb, p=p, dt=dt: {"prod": (rb.fromarray(p).prod(), want_prod(p, dt), "bits")})
    for kind in ("decades", "cancel"):
        b = family_b(min(n1, 1 << 22), 16, kind)
        add("b_sum_%s" % kind, "kernel=stream mode=elementwise",
            lambda rb, b=b: {"sum": (rb.fromarray(b).sum(), None, ("ratio", chain_global(b.size), b))})
        add("b_axis_sum_%s" % kind, AXIS_SPLIT,
            lambda rb, b=b: {"sum": (rb.fromarray(b[: (b.size // 37) * 37].reshape(-1, 37)).sum(axis=0)[5], None,
                                     ("ratio", chain_global(b.size // 37), b[: (b.size // 37) * 37].reshape(-1, 37)[:, 5]))})
        bs = b[: 1 << 20]
        add("b_cumsum_%s" % kind, "kernel=scan form=lookback", lambda rb, bs=bs: {"cumsum": (rb.cumsum(rb.fromarray(bs)), None, ("cratio", chain_scan(bs.size), bs))})
    for dt in (onp.float32, onp.float64):  # nansum / nanmean on family A data with NaN holes
        tag = "f32" if dt == onp.float32 else "f64"
        x, ints, e0 = family_a((n1,), dt, 17)
        hole = onp.zeros(n1, dtype=bool)
        hole[::7] = True
        xn = x.copy()
        xn[hole] = onp.nan
        s_nan = round_to(ints[~hole].sum(), e0, dt)
        add("nansum_%s" % tag, "kernel=general_interpreter form=elementwise", lambda rb, xn=xn, s_nan=s_nan: {"nansum": (rb.nansum(rb.fromarray(xn)), s_nan, "bits")})
        add("nanmean_%s" % tag, "kernel=general_interpreter form=elementwise", lambda rb, xn=xn, s_nan=s_nan, k=int((~hole).sum()): {
            "nanmean": (onp.float64(rb.nanmean(rb.fromarray(xn))), onp.float64(s_nan / onp.int64(k)), "bits")})
    pb = onp.random.default_rng(18).uniform(0.5, 2.0, 4099)
    add("b_prod", "kernel=stream mode=elementwise", lambda rb, pb=pb: {"prod": (rb.fromarray(pb).prod(), None, ("pratio", chain_any(pb.size), pb))})
    for gname, shape, dim, G, gform in GROUP_CASES:
        for dt in (onp.float32, onp.float64):
            g, _, _ = family_a(shape, dt, 19 + G)
            labels = onp.random.default_rng(G).integers(0, G, shape[dim])
            add("group_%s_%s" % (gname, dt.__name__), gform, lambda rb, g=g, dim=dim, G=G, labels=labels, dt=dt: _group_sums(rb, g, dim, G, labels, dt))
    gv = 1e8 + onp.random.default_rng(23).standard_normal((8 if big else 4, 1 << 18 if big else 20000))
    add("group_var_offset", "kernel=group form=row", lambda rb, gv=gv: _group_var(rb, gv))
    # specials
    add("specials", ("kernel=stream mode=elementwise", "kernel=general_interpreter form=axis_reduce", "kernel=reduce_partials",
                     "kernel=scan form=lookback", "kernel=scan form=columns"), _specials)
    add("nan_minmax", ("kernel=mapred mode=global", "kernel=stream mode=elementwise", "kernel=general_interpreter form=axis_reduce",
                       "kernel=reduce_partials", "kernel=scan form=lookback"), lambda rb: _nan_minmax(rb, n1))
    return cases


# the split axis form: the interpreter's axis reduction into per-split partials, folded by reduce_partials
AXIS_SPLIT = ("kernel=general_interpreter form=axis_reduce", "kernel=reduce_partials")

# (name, shape, grouped axis, groups, group plan the case must reach): every form of the grouped-reduction kernel
GROUP_CASES = [
    ("row_split", (5, 20000), 1, 3, lambda p: p.startswith("kernel=group form=row") and " chunks=1 " not in p),
    ("general", (20000, 3), 0, 2, "kernel=group form=general"),
    ("column", (3000, 64), 0, 2, "kernel=group form=column"),
    ("many_groups", (10, 3000), 1, 2000, "kernel=group form=general"),
]


def _group_members(labels, G):
    return [onp.flatnonzero(labels == g) for g in range(G)]


def _group_sums(rb, x, dim, G, labels, dt):
    """groupby sum (result dtype), mean and nanmean (float64) on family A data: the exact group sums, rounded once;
    the means are the float64 sum (exact) divided by the count, one rounding."""
    ints, e = exact_ints(x)
    xi = onp.moveaxis(ints, dim, -1)
    sums = onp.stack([xi[..., m].sum(axis=-1) for m in _group_members(labels, G)], axis=-1)
    cnt = onp.bincount(labels, minlength=G).astype(onp.float64)
    want_s = onp.moveaxis(round_to(sums, e, dt), -1, dim)
    with onp.errstate(all="ignore"):
        want_m = onp.moveaxis(round_to(sums, e, onp.float64) / cnt, -1, dim)
    gb = rb.fromarray(x).groupby(dim, labels, G)
    return {"sum": (gb.sum(), want_s, "bits"), "mean": (gb.mean(), want_m, "bits"), "nanmean": (gb.nanmean(), want_m, "bits")}


def var_bound(x, d):
    """(exact variance, bound on |got - exact|) of one group for the two-pass SQDEV form: the centre c = fl(fl(S) / m) is
    off the exact mean mu by at most delta = u |mu| + gamma_d sum|x| / m; x - c is exact (Sterbenz: c and x within a
    factor 2 of each other), so the accumulated sum(fl((x - c)^2)) is (sum (x - mu)^2 + m delta^2)(1 + theta) with
    |theta| <= gamma_{d+1}, and the division by m adds one rounding."""
    m = len(x)
    fr = [Fraction(float(v)) for v in x]
    mu = sum(fr) / m
    var = sum((v - mu) ** 2 for v in fr) / m
    delta = Fraction(U64) * abs(mu) + Fraction(gamma(d)) * sum(abs(v) for v in fr) / m
    assert all(float(c) / 2 <= v <= 2 * float(c) for c in (mu,) for v in x)
    return var, delta ** 2 + Fraction(gamma(d + 2)) * (var + delta ** 2)


def var_one_pass(x):
    """The rejected form: E[x^2] - E[x]^2 in float64."""
    x = onp.asarray(x, dtype=onp.float64)
    return (x * x).mean() - x.mean() ** 2


def _group_var(rb, x):
    """groupby var / std along axis 1 (two groups per row) of 1e8 + noise: within var_bound of the exact rational
    variance, and its square root."""
    labels = onp.arange(x.shape[1]) % 2
    gb = rb.fromarray(x).groupby(1, labels, 2)
    var, std = onp.asarray(gb.var().asarray()), onp.asarray(gb.std().asarray())
    worst = 0.0
    for i in range(x.shape[0]):
        for g in range(2):
            xs = x[i, labels == g]
            exact, bound = var_bound(xs, chain_any(xs.size))
            worst = max(worst, float(abs(Fraction(float(var[i, g])) - exact) / bound))
            lo, hi = math.sqrt(float(exact - bound)) * (1 - 2 * U64), math.sqrt(float(exact + bound)) * (1 + 2 * U64)
            assert lo <= std[i, g] <= hi, (i, g, std[i, g], lo, hi)
    return {"var": (worst, None, ("given",))}


def _specials(rb):
    out = {}
    r = onp.random.default_rng(20)
    for dt in (onp.float32, onp.float64):
        for what, vals in (("nan", [onp.nan]), ("infs", [onp.inf, -onp.inf]), ("inf", [onp.inf]), ("ninf", [-onp.inf])):
            x = r.uniform(-1, 1, 10007).astype(dt)
            x[r.choice(x.size, size=len(vals), replace=False)] = vals
            out["sum_%s_%s" % (what, dt.__name__)] = (rb.fromarray(x).sum(), x.sum(), "bits")
            out["cumsum_last_%s_%s" % (what, dt.__name__)] = (rb.cumsum(rb.fromarray(x)).asarray()[-1:], onp.cumsum(x)[-1:], "bits")
        z = onp.full(5003, -0.0, dtype=dt)
        out["sum_negzero_%s" % dt.__name__] = (onp.signbit(onp.asarray(rb.fromarray(z).sum())), onp.signbit(z.sum()), "bits")
        out["cumsum_negzero_%s" % dt.__name__] = (onp.signbit(rb.cumsum(rb.fromarray(z)).asarray()), onp.signbit(onp.cumsum(z)), "bits")
        z2 = onp.full((70, 33), -0.0, dtype=dt)
        out["cumsum_cols_negzero_%s" % dt.__name__] = (onp.signbit(rb.cumsum(rb.fromarray(z2), axis=0).asarray()),
                                                       onp.signbit(onp.cumsum(z2, axis=0)), "bits")
        x = onp.full(4099, 1.0, dtype=dt)
        x[::2] = onp.nan
        out["nansum_%s" % dt.__name__] = (rb.nansum(rb.fromarray(x)), onp.nansum(x), "bits")
        out["nanmean_%s" % dt.__name__] = (onp.float64(rb.nanmean(rb.fromarray(x))), onp.float64(onp.nanmean(x)), "bits")
    big = onp.full(4099, 3e38, dtype=onp.float32)
    out["sum_overflow_f32"] = (rb.fromarray(big).sum(), onp.float32(onp.inf), "bits")
    out["axis_sum_overflow_f32"] = (rb.fromarray(big.reshape(1, -1)).sum(axis=1), onp.full(1, onp.inf, dtype=onp.float32), "bits")
    return out


def nan_positions(n):
    """One NaN per position class: first / last element of a thread's group and of a 16 x 256 or 2048 tile, the two
    halves of an in-thread tree step, another CTA, the ragged tail, the last element."""
    ps = {0, 1, 3, 4, 7, 8, 15, 16, 255, 256, 2047, 2048, 4095, 4096, n // 2, n // 3 + 1, n - (n % 4096) + 1, n - 2, n - 1}
    return sorted(p for p in ps if 0 <= p < n)


def _nan_minmax(rb, n):
    out = {}
    r = onp.random.default_rng(21)
    base = r.uniform(-1, 1, n)
    for dt in (onp.float32, onp.float64):
        for p in nan_positions(n):
            x = base.astype(dt)
            x[p] = onp.nan
            A = rb.fromarray(x)
            for op in ("min", "max"):
                out["%s_%s_%d" % (op, dt.__name__, p)] = (getattr(A, op)(), getattr(onp, op)(x), "bits")
        x = base.astype(dt)
        x[r.integers(0, n)] = onp.nan
        A = rb.fromarray(x)
        out["map_min_%s" % dt.__name__] = ((A * 2.0 + 1.0).min(), (x * dt(2.0) + dt(1.0)).min(), "bits")
        m = base[: (n // 37) * 37].reshape(-1, 37).astype(dt)
        m[m.shape[0] // 2, 3] = onp.nan
        m[0, 5] = onp.nan
        m[-1, 7] = onp.nan
        M = rb.fromarray(m)
        for op in ("min", "max"):
            for ax in (0, 1):
                out["%s_axis%d_%s" % (op, ax, dt.__name__)] = (getattr(M, op)(axis=ax), getattr(onp, op)(m, axis=ax), "bits")
            out["scumulative_%s_%s" % (op, dt.__name__)] = (
                rb.scumulative(getattr(onp, "minimum" if op == "min" else "maximum"), getattr(onp, "minimum" if op == "min" else "maximum"),
                               rb.fromarray(x)).asarray(), (onp.minimum if op == "min" else onp.maximum).accumulate(x), "bits")
        allnan = onp.full(5000, onp.nan, dtype=dt)
        out["min_allnan_%s" % dt.__name__] = (rb.fromarray(allnan).min(), onp.min(allnan), "bits")
        out["max_allnan_%s" % dt.__name__] = (rb.fromarray(allnan).max(), onp.max(allnan), "bits")
    return out


def _value(v):
    import ramba_b200 as rb

    return onp.asarray(v.asarray() if isinstance(v, rb.ndarray) else v)


def evaluate(size, only=None):
    """Run every case: ({case: {label: [n_bad or ratio, kind]}}, {case: [plan prefixes of its op lists]})."""
    import ramba_b200 as rb
    from ramba_b200 import _cabi
    from ramba_b200.runtime import RT

    results, plans = {}, {}
    for name, form, build in _cases(size):
        if only is not None and name not in only:
            continue
        be = RT.be()
        run = be.run
        seen = []

        def record(fop, stream=None):
            seen.append(_cabi.describe_plan(fop))
            return run(fop, stream)

        def scan(src, dst, code, n_outer, length, n_inner, *a, **k):
            # the library picks the look-back kernel exactly when the scan axis is innermost (n_inner == 1)
            seen.append("kernel=scan form=%s" % ("lookback tiles=%d" % (n_outer * -(-length // 2048)) if n_inner == 1 else "columns"))
            return cumulative(src, dst, code, n_outer, length, n_inner, *a, **k)

        def partials(out, part, n, k, *a):
            seen.append("kernel=reduce_partials splits=%d" % k)
            return reduce_partials(out, part, n, k, *a)

        def group(view, code, axis, table, *a):
            seen.append(_cabi.describe_group_plan(view, axis, table.n_groups))
            return group_reduce(view, code, axis, table, *a)

        cumulative, reduce_partials, group_reduce = RT.cumulative, RT.reduce_partials, RT.group_reduce
        be.run, RT.cumulative, RT.reduce_partials, RT.group_reduce = record, scan, partials, group
        try:
            got = build(rb)
            vals = {k: (_value(g), w, kind) for k, (g, w, kind) in got.items()}
            rb.sync()
        finally:
            be.run = run
            del RT.cumulative, RT.reduce_partials, RT.group_reduce
        res = {}
        for label, (g, w, kind) in vals.items():
            if kind == "bits":
                res[label] = [same_bits(g, onp.asarray(w)), "bits"]
            elif kind[0] == "ratio":
                res[label] = [sum_error_ratio(g, kind[2], kind[1]), "ratio"]
            elif kind[0] == "pratio":
                res[label] = [prod_error_ratio(g, kind[2], kind[1]), "ratio"]
            elif kind[0] == "given":
                res[label] = [float(g), "ratio"]
            else:
                res[label] = [cumsum_error_ratio(g, kind[2], kind[1]), "ratio"]
        results[name] = res
        print("case %s done" % name, file=sys.stderr, flush=True)
        plans[name] = seen
        del got, vals
    return results, plans


def check(results, plans, size, forms=True):
    forms = {name: (form if forms else None) for name, form, _ in _cases(size)}
    report = {}
    for name, res in results.items():
        for label, (v, kind) in res.items():
            if kind == "bits":
                assert v == 0, (name, label, v, plans[name])
            else:
                assert v <= 1.0, (name, label, v)
                report[name] = max(report.get(name, 0.0), v)
        if forms[name] is not None:
            for f in forms[name] if isinstance(forms[name], tuple) else (forms[name],):
                hit = f if callable(f) else (lambda p, f=f: p.startswith(f))
                assert any(hit(p) for p in plans[name]), (name, f, plans[name])
    return report


def test_oracle_cases(oracle_engine):
    results, plans = evaluate("small")
    report = check(results, plans, "small")
    print("err/bound (oracle):", json.dumps(report, indent=1))


def test_nan_min_max_on_the_oracle_is_numpy(oracle_engine):
    import ramba_b200 as rb

    x = onp.arange(20.0).reshape(4, 5)
    x[1, 2] = onp.nan
    a = rb.fromarray(x)
    assert math.isnan(a.max()) and math.isnan(a.min())
    assert_bits(a.max(axis=0).asarray(), x.max(axis=0))
    assert math.isnan((a * 2.0 + 1.0).min())
    assert math.isnan(rb.fromarray(onp.array([1.0, onp.nan, 2.0, 0.5])).min())


# ---- several ranks ------------------------------------------------------------------------------------------------------
SUMS_1D = [("sum", None), ("cumsum", 0)]
SUMS_2D = [("sum", 0), ("sum", 1), ("sum", None), ("cumsum", 0), ("cumsum", 1)]
MINMAX_1D = [("min", None), ("max", None)]
MINMAX_2D = [("min", 0), ("max", 0), ("min", 1), ("max", 1), ("min", None), ("max", None)]


def world_sources():
    """(name, array, [(op, axis)]) of the world programs: every rank builds the same values."""
    out = []
    r = onp.random.default_rng(32)
    for dt in (onp.float32, onp.float64):
        tag = "f32" if dt == onp.float32 else "f64"
        x, _, _ = family_a((40009,), dt, 30)
        out.append(("v_%s" % tag, x, SUMS_1D + MINMAX_1D))
        m, _, _ = family_a((3001, 7), dt, 31)
        out.append(("m_%s" % tag, m, SUMS_2D))
        for p in (0, 1999, 4000):  # on the first, a middle and the last rank
            y = r.uniform(-1, 1, 4001).astype(dt)
            y[p] = onp.nan
            out.append(("nan%d_%s" % (p, tag), y, MINMAX_1D))
        y = r.uniform(-1, 1, (1001, 5)).astype(dt)
        y[[0, 500, 1000], [1, 2, 3]] = onp.nan
        out.append(("nan2d_%s" % tag, y, MINMAX_2D))
        out.append(("scan_nan_%s" % tag, y[:, 1].copy(), [("scummin", 0), ("scummax", 0)]))
        out.append(("negzero_%s" % tag, onp.full(4001, -0.0, dtype=dt), [("cumsum", 0), ("sum", None)]))
        out.append(("negzero2d_%s" % tag, onp.full((4001, 3), -0.0, dtype=dt), [("cumsum", 0), ("cumsum", 1)]))
    return out


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
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_accum_worker.py"), out, mode], env=env,
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


def f32_world_model(x, blocks, axis):
    """float32 sum at W ranks: each rank's block sum rounded to float32 (the partial array has the result dtype), the
    rank partials added exactly (float64 all-reduce of a few float32 values) and rounded to float32 once more."""
    nd = x.ndim
    ints, e = exact_ints(x)
    tot = None
    for b in blocks:
        st, sz = b[:nd], b[nd:]
        if (sz == 0).any():
            continue
        sl = tuple(slice(int(s), int(s) + int(z)) for s, z in zip(st, sz))
        part = round_to(ints[sl].sum(axis=axis), e, onp.float32).astype(onp.float64)
        if axis is not None:
            full = onp.zeros(onp.delete(onp.array(x.shape), axis), dtype=onp.float64)
            keep = tuple(s for d, s in enumerate(sl) if d != axis)
            full[keep] = part
            part = full
        tot = part if tot is None else tot + part
    return onp.asarray(tot).astype(onp.float32)


def _expected_world(name, x, op, axis, blocks, world):
    dt = x.dtype.type
    if op in ("scummin", "scummax"):
        return (onp.minimum if op == "scummin" else onp.maximum).accumulate(x, axis=axis)
    if name.startswith("negzero"):
        return onp.cumsum(x, axis=axis) if op == "cumsum" else x.sum(axis=axis)
    if op == "cumsum":
        return want_cumsum(x, dt, axis)
    if op in ("min", "max"):
        return getattr(onp, op)(x, axis=axis)
    if dt == onp.float64 or world == 1:
        return want_sum(x, dt, axis)
    return f32_world_model(x, blocks, axis)


@pytest.fixture(scope="module")
def accum_worlds(tmp_path_factory):
    d = tmp_path_factory.mktemp("accum_worlds")
    return {w: _run_world(w, str(d / ("w%d.npz" % w))) for w in (1, 2, 3, 4, 8)}


@pytest.mark.timeout(1800)
def test_worlds_match_one_rank_and_the_exact_model(accum_worlds):
    base = accum_worlds[1]
    split = 0
    for w, res in accum_worlds.items():
        for name, x, ops in world_sources():
            blocks = res[name + ".blocks"]
            split += int(w > 1 and (blocks[:, x.ndim:] > 0).all(axis=1).sum() > 1)
            for op, axis in ops:
                key = "%s.%s.%s" % (name, op, axis)
                got = res[key]
                assert_bits(got, _expected_world(name, x, op, axis, blocks, w), "W=%d %s" % (w, key))
                if x.dtype == onp.float64 or op != "sum":
                    assert_bits(got, base[key], "W=%d %s against W=1" % (w, key))
    assert split > 0


# ---- GPU ----------------------------------------------------------------------------------------------------------------
SWITCHES = {"default": {}, "no_mapred": {"RB200_NO_MAPRED_KERNEL": "1"}, "no_stream": {"RB200_NO_STREAM_KERNEL": "1"},
            "no_terms": {"RB200_NO_TERMS_KERNEL": "1"}, "no_lean": {"RB200_NO_LEAN_INTERP": "1"}}
# what each switch set must keep every op list off
BARRED = {"no_mapred": lambda p: p.startswith("kernel=mapred"), "no_stream": lambda p: p.startswith("kernel=stream "),
          "no_terms": lambda p: p.startswith("kernel=stream_terms"), "no_lean": lambda p: p.endswith("variant=lean")}


def check_switched(switches, results, plans, size):
    """Numbers as check(); the named forms under the default switches, and no op list on a barred kernel otherwise."""
    if switches == "default":
        return check(results, plans, size)
    bar = BARRED[switches]
    for name, ps in plans.items():
        assert not any(bar(p) for p in ps), (switches, name, ps)
    return check(results, {k: [] for k in plans}, size, forms=False)


def _plans_worker(out_dir, switches):
    """The small cases on the oracle backend in a process of their own (the switches are read once per process)."""
    from ramba_b200.runtime import RT

    RT.reset()
    if switches != "gpu":
        import _oracle_backend

        _oracle_backend.install()
    elif os.environ.get("RB200_DRY_GPU_TESTS"):
        import conftest

        conftest._dry_gpu()
    with onp.errstate(all="ignore"):
        results, plans = evaluate("small" if switches != "gpu" else os.environ["RB200_ACCUM_SIZE"])
    with open(os.path.join(out_dir, "out.json"), "w") as f:
        json.dump([results, plans], f)


def _run_switched(tmp_path, switches, backend, size="small"):
    code = "import sys; sys.path[:0] = [%r, %r]; import test_reduction_accuracy as t; t._plans_worker(%r, %r)" % (
        ROOT, HERE, str(tmp_path), "gpu" if backend == "gpu" else switches)
    env = dict(os.environ, RB200_ACCUM_SIZE=size, **SWITCHES[switches])
    out = subprocess.run([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, text=True, timeout=3000)
    assert out.returncode == 0, out.stdout[-2000:]
    with open(os.path.join(str(tmp_path), "out.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("switches", [s for s in SWITCHES if s != "default"])
def test_switched_kernels_on_the_oracle(tmp_path, switches):
    results, plans = _run_switched(tmp_path, switches, "oracle")
    check_switched(switches, results, plans, "small")


@pytest.mark.gpu
@pytest.mark.timeout(3600)
@pytest.mark.parametrize("switches", list(SWITCHES))
def test_accumulation_on_the_gpu(tmp_path, switches):
    size = "big" if switches == "default" else "small"
    results, plans = _run_switched(tmp_path, switches, "gpu", size)
    report = check_switched(switches, results, plans, size)
    print("err/bound (%s):" % switches, json.dumps(report, indent=1))


@pytest.mark.gpu
@pytest.mark.timeout(1200)
def test_float32_sum_past_2_31_elements(gpu_engine):
    """One float32 global sum over 2^31 + 4097 elements (8.6 GB): x_i = ((i * 40503) mod 2^16 - 2^15) * 2^-20.  Partial
    sums reach 2^31 * 2^-20, far past float32's 24 bits, and stay exact in float64.  40503 is odd, so every full period
    of 2^16 indices sums to -2^15; the ragged remainder is summed on the host."""
    import ramba_b200 as rb

    n, period, a = (1 << 31) + 4097, 1 << 16, 40503
    X = (((rb.arange(n) * a) % period - period // 2) * 2.0 ** -20).astype(onp.float32)
    rb.sync()
    reps = n // period
    rem = (onp.arange(reps * period, n, dtype=onp.int64) * a) % period - period // 2
    exact = -(period // 2) * reps + int(rem.sum())
    want = onp.float32(onp.ldexp(float(exact), -20))
    assert_bits(onp.asarray(X.sum()), want, "2^31 + 4097 float32 sum")
