"""Integer and truth reductions and scans, held to exact Python-integer references.

The contract (DESIGN §6), each result bit for bit:

  * sum / prod of integer and bool data keep the input dtype and wrap: the exact Python-int total reduced modulo 2^bits
    into the dtype (wrapping is a ring homomorphism, so every order of summation gives the same bits); for bool, sum is
    any and prod is all.
  * min / max: the integers' min / max.  all / any: Python all / any over x != 0 (NaN is true, -0.0 is false).
  * mean / nanmean of integer and bool data: NumPy's float64 sum of float64(x) divided by n.  The data keep every float64
    partial exact, so the global form is Fraction(sum, n) correctly rounded; the axis form is s * (1.0 / n), within 1 ulp.
  * sum / prod(dtype=D): each element is converted to D first.
  * cumsum of integer and bool data: int64, the exact prefix sums modulo 2^64 (NumPy gives uint64 for unsigned input:
    a kept deviation).  scumulative min / max / prod and groupby sum / prod / min / max / count / mean: the same models.

Uniform small integers cannot tell a wrong accumulator from a right one, so the data are where it shows: full-range
values whose totals wrap (odd values near +-2^62 for int64: a float64 accumulator anywhere loses the low bits), odd
factors only (the wrapped product never collapses to 0), the extremes of each width and unsigned values with the top bit
set at every position class, cancelling pairs for any, wrapping / underflowing products for all.

The CPU tests run the engine on the oracle backend, over gloo worlds of 1 to 8 ranks, and show that each check fails on
a deliberately wrong host restatement.  The GPU tests run the same cases on the kernels, each case asserting through
rb200_describe_plan the form it reaches, in one process per set of kernel switches (RB200_NO_*)."""
import builtins as builtins_mod
import json
import os
import subprocess
import sys
from fractions import Fraction

import numpy as onp
import pytest

import test_reduction_accuracy as T

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

INTS = (onp.int64, onp.int32, onp.int16, onp.int8, onp.uint32, onp.uint16, onp.uint8)
DTYPES = INTS + (onp.bool_,)
same_bits, assert_bits = T.same_bits, T.assert_bits


# ---- exact models -------------------------------------------------------------------------------------------------------
def bits_of(dt):
    return 1 if dt == onp.bool_ else onp.dtype(dt).itemsize * 8


def wrap(v, dt):
    """Python int v reduced modulo 2^bits into dtype dt (bool: v != 0)."""
    v = int(v)
    if dt == onp.bool_:
        return onp.bool_(v != 0)
    b = bits_of(dt)
    v &= (1 << b) - 1
    if onp.issubdtype(dt, onp.signedinteger) and v >= 1 << (b - 1):
        v -= 1 << b
    return onp.dtype(dt).type(v)


def exact_total(x, axis=None):
    """Exact Python-int sum of integer data (any shape, fewer than 2^31 elements along the reduced axes): the high and
    low 32-bit halves are summed separately, each without overflow in int64."""
    x = onp.asarray(x).astype(onp.int64)
    hi, lo = x >> 32, x & 0xFFFFFFFF
    sh, sl = hi.sum(axis=axis), lo.sum(axis=axis)
    if axis is None:
        return (int(sh) << 32) + int(sl)
    return onp.array([(int(a) << 32) + int(b) for a, b in zip(sh.reshape(-1), sl.reshape(-1))], dtype=object).reshape(sh.shape)


def want_sum(x, axis=None):
    dt = x.dtype.type
    t = exact_total(x, axis)
    if axis is None:
        return wrap(t, dt)
    return onp.array([wrap(v, dt) for v in t.reshape(-1)], dtype=dt).reshape(t.shape)


def exact_prod(x):
    p = 1
    for v in onp.asarray(x).reshape(-1).tolist():
        p = (p * int(v)) & ((1 << 64) - 1)  # (modulo 2^64 keeps every narrower residue)
    return p


def want_prod(x):
    return wrap(exact_prod(x), x.dtype.type)


def want_mean(x, axis=None):
    """Global: Fraction(sum, n) correctly rounded.  Axis: the engine's s * (1.0 / n) on the exact float64 sums, checked
    here to lie within 1 ulp of the exact quotient."""
    t = exact_total(x, axis)
    if axis is None:
        assert abs(t) < 2 ** 53
        return onp.float64(float(Fraction(t, x.size)))
    n = x.shape[axis]
    s = onp.array([float(v) for v in t.reshape(-1)])
    assert (onp.abs(s) < 2 ** 53).all()
    m = s * (1.0 / n)
    exact = onp.array([float(Fraction(int(v), n)) for v in t.reshape(-1)])
    assert (onp.abs(m - exact) <= onp.spacing(onp.abs(exact))).all()
    return m.reshape(t.shape)


def want_cumsum(x, axis):
    """int64 prefix sums modulo 2^64 (high and low halves scanned separately in int64, then joined modulo 2^64)."""
    x = onp.asarray(x).astype(onp.int64)
    ch, cl = onp.cumsum(x >> 32, axis=axis), onp.cumsum(x & 0xFFFFFFFF, axis=axis)
    return ((ch.astype(onp.uint64) << onp.uint64(32)) + cl.astype(onp.uint64)).view(onp.int64)


def want_cumprod(x):
    out = onp.empty(x.size, dtype=onp.int64)
    p = 1
    for i, v in enumerate(x.reshape(-1).tolist()):
        p = (p * int(v)) & ((1 << 64) - 1)
        out[i] = p - (1 << 64) if p >= 1 << 63 else p
    return out


def truth(x):
    """Python all / any see x != 0: NaN is true, -0.0 is false."""
    return [bool(v != 0) for v in onp.asarray(x).reshape(-1).tolist()]


# ---- data where the accumulator shows -----------------------------------------------------------------------------------
def full_range(n, dt, seed):
    """Full-range values; for int64, odd values near +-2^62, so the total wraps past 2^63 several times and has every low
    bit set somewhere."""
    r = onp.random.default_rng(seed)
    if dt == onp.bool_:
        return r.random(n) < 0.5
    if dt == onp.int64:
        v = (onp.int64(1) << onp.int64(62)) - r.integers(0, 1 << 40, size=n, dtype=onp.int64)
        return (v | 1) * r.choice(onp.array([-1, 1], dtype=onp.int64), size=n)
    info = onp.iinfo(dt)
    return r.integers(int(info.min), int(info.max), size=n, endpoint=True, dtype=onp.int64).astype(dt)


def odd_factors(n, dt, seed):
    """Odd factors of either sign below min(2^20, the dtype's max): the wrapped product is odd, so never 0, and every
    dropped or doubled factor changes it."""
    r = onp.random.default_rng(seed)
    if dt == onp.bool_:
        return onp.ones(n, dtype=bool)
    hi = min(1 << 20, int(onp.iinfo(dt).max))
    v = r.integers(0, (hi - 1) // 2, size=n, dtype=onp.int64) * 2 + 1
    if onp.issubdtype(dt, onp.signedinteger):
        v *= r.choice(onp.array([-1, 1], dtype=onp.int64), size=n)
    return v.astype(dt)


def mean_data(shape, dt, seed):
    """Integer data whose float64 sums are exact in every order (|sum| < 2^53)."""
    r = onp.random.default_rng(seed)
    if dt == onp.bool_:
        return r.random(shape) < 0.7
    n = int(onp.prod(shape))
    lim = min(int(onp.iinfo(dt).max), (1 << 52) // n)
    lo = 0 if onp.issubdtype(dt, onp.unsignedinteger) else -lim
    v = r.integers(lo, lim, size=shape, endpoint=True, dtype=onp.int64)
    if dt != onp.int64:
        v[..., 0] = int(onp.iinfo(dt).max)  # the narrow sum wraps
    return v.astype(dt)


def positions(n):
    """Position classes: first / last element, each element slot of a thread's 16, CTA and tile edges (256, 2048, 4096),
    a middle element, the ragged last tile and the last element."""
    return sorted(set(T.nan_positions(n)) | set(range(16)) | {4096 + 8, 2048 + 15})


def minmax_data(n, dt, seed, which, p):
    """`which` ("min" / "max") at position p is the extreme of the width; the rest are values that expose a
    sign-extending load (unsigned: top bit set for min, clear for max) or a narrower identity (int64: beyond int32)."""
    r = onp.random.default_rng(seed)
    info = onp.iinfo(dt)
    b = bits_of(dt)
    if onp.issubdtype(dt, onp.unsignedinteger):
        x = r.integers(1 << (b - 1), (1 << b) - 1, size=n, dtype=onp.int64) if which == "min" else r.integers(0, 1 << (b - 1), size=n, dtype=onp.int64)
    else:
        x = r.integers(int(info.min) + 1, int(info.max), size=n, dtype=onp.int64)
    x = x.astype(dt)
    x[p] = info.min if which == "min" else info.max
    return x


def wide_minmax(n, which, dt, seed):
    """No extreme present: int64 values all above 2^32 (min) or all below -2^32 (max), uint32 all at or above 2^31 (min):
    an int32-width identity or a signed 32-bit compare gives a wrong answer."""
    r = onp.random.default_rng(seed)
    if dt == onp.uint32:
        return r.integers(1 << 31, 1 << 32, size=n, dtype=onp.int64).astype(onp.uint32)
    v = r.integers(1 << 32, 1 << 62, size=n, dtype=onp.int64)
    return v if which == "min" else -v


# ---- deliberately wrong host restatements (each check must fail on them) ------------------------------------------------
def restated_sum(x, acc=onp.int64, drop=False, double_partial=False, cta=256):
    """Sum in the shape of the kernels: one partial per CTA of `cta` elements, then the fold of the partials, stored to
    x's dtype.  acc: accumulator dtype; drop: lose the last element; double_partial: fold the second partial twice."""
    x = onp.asarray(x).reshape(-1)
    if drop:
        x = x[:-1]
    parts = [x[i:i + cta].astype(acc).sum(dtype=acc) for i in range(0, x.size, cta)]
    if double_partial and len(parts) > 1:
        parts.append(parts[1])
    tot = acc(0)
    with onp.errstate(all="ignore"):
        for p in parts:
            tot = acc(tot + p)
    return wrap(int(tot), x.dtype.type)


def test_each_check_fails_on_a_wrong_restatement():
    # sums: the int64 accumulator matches the model, a float64 one, a dropped element and a doubled partial do not
    for dt in INTS:
        x = full_range(10007, dt, 1)
        assert_bits(restated_sum(x), want_sum(x), dt)
        for wrong in (dict(acc=onp.float64), dict(drop=True), dict(double_partial=True)):
            if wrong.get("acc") == onp.float64 and dt != onp.int64:
                continue  # (a narrow total is exact in float64 at this size; int64 data are where it shows)
            assert same_bits(restated_sum(x, **wrong), want_sum(x)) > 0, (dt, wrong)
    # products of odd factors: a dropped or doubled factor changes the wrapped product
    for dt in INTS:
        x = odd_factors(4099, dt, 2)
        assert int(want_prod(x)) % 2 == 1
        assert same_bits(want_prod(x[:-1]), want_prod(x)) > 0 and same_bits(want_prod(onp.append(x, x[7])), want_prod(x)) > 0
    # any as a wrapping sum, all as a product
    for dt in INTS:
        x = any_cancel(4099, dt)
        assert any(truth(x))
        assert not wrap(exact_total(x), dt)
        y = all_wrap(4099, dt)
        assert all(truth(y)) and not wrap(exact_prod(y), onp.int64)
    for dt, tiny, huge in ((onp.float64, 1e-200, 1e308), (onp.float32, 1e-30, 3e38)):
        with onp.errstate(all="ignore"):
            assert onp.prod(onp.array([tiny, tiny], dtype=dt)) == 0 and all(truth(onp.array([tiny, tiny], dtype=dt)))
            assert onp.prod(onp.array([onp.nan, 0.0], dtype=dt)) != 0 and not all(truth(onp.array([onp.nan, 0.0], dtype=dt)))
            assert onp.prod(onp.array([huge, -huge, 0.0], dtype=dt)) != 0
            assert onp.sum(onp.array([0.5, -0.5], dtype=dt)) == 0 and any(truth(onp.array([0.5, -0.5], dtype=dt)))
    assert not any(truth(onp.array([-0.0, -0.0])))
    # mean over the wrapped sum
    for dt in INTS[1:] + (onp.bool_,):
        x = mean_data((4099,), dt, 3)
        wrapped = onp.float64(int(want_sum(x))) / x.size
        assert same_bits(wrapped, want_mean(x)) > 0, dt
    # a float64 accumulator for int64 loses the low bits; a sign-extending uint32 load changes the int64 prefix sums,
    # sum(dtype=int64) and the max (a wrapped uint32 sum is the same either way)
    x = full_range(10007, onp.int64, 4)
    assert same_bits(restated_sum(x, acc=onp.float64), want_sum(x)) > 0
    u = minmax_data(4099, onp.uint32, 5, "max", 100)
    assert same_bits(want_cumsum(u.view(onp.int32), 0), want_cumsum(u, 0)) > 0
    assert exact_total(u.view(onp.int32)) != exact_total(u)
    assert onp.uint32(u.view(onp.int32).max()) != onp.uint32(u.max())
    um = minmax_data(4099, onp.uint32, 5, "min", 100)
    assert onp.uint32(um.view(onp.int32).min()) != onp.uint32(um.min())
    # an int32-width identity for min / max
    for which in ("min", "max"):
        w = wide_minmax(4099, which, onp.int64, 6)
        ident = (1 << 31) - 1 if which == "min" else -(1 << 31)
        assert getattr(builtins_mod, which)(ident, *w.tolist()) != getattr(builtins_mod, which)(w.tolist())
    # cumsum: a 32-bit accumulator for int32 / uint32 data differs once the prefixes pass 2^32
    s = full_range(70001, onp.uint32, 7)
    assert same_bits(onp.cumsum(s, dtype=onp.uint32).astype(onp.int64), want_cumsum(s, 0)) > 0



def any_cancel(n, dt):
    """Zeros plus pairs (x, -x) (unsigned: x, 2^bits - x), whose sum is 0 in the dtype."""
    x = onp.zeros(n, dtype=onp.int64)
    b = bits_of(dt)
    v = 3 if b > 8 else 5
    x[1], x[n - 2] = v, (-v if onp.issubdtype(dt, onp.signedinteger) else (1 << b) - v)
    x[n // 2], x[n // 2 + 1] = 2, (-2 if onp.issubdtype(dt, onp.signedinteger) else (1 << b) - 2)
    return x.astype(dt)


def all_wrap(n, dt):
    """Ones and 64 or more twos (-2 in signed types), whose product wraps to 0 modulo 2^64."""
    x = onp.ones(n, dtype=onp.int64)
    x[onp.linspace(0, n - 1, 70).astype(onp.int64)] = -2 if onp.issubdtype(dt, onp.signedinteger) else 2
    return x.astype(dt)


# ---- engine cases, shared by the oracle and the GPU tests ---------------------------------------------------------------
INTERP = "kernel=general_interpreter"
ELEMENTWISE = INTERP + " form=elementwise"


def _cases(size):
    """[(name, form, build(rb) -> {label: (got, want)})]: every result bit for bit; form as in test_reduction_accuracy."""
    big = size == "big"
    n1 = (1 << 24) + 12345 if big else 100003
    npos = 100003                                    # the position-class arrays (one array per position)
    nscan = 2400 * 2048 + 4099 if big else 70001
    rows = (1 << 18) + 7 if big else 4099
    cases = []

    def add(name, form, fn):
        cases.append((name, form, fn))

    for dt in DTYPES:
        tag = onp.dtype(dt).name
        x = full_range(n1, dt, 10)
        add("sum_%s" % tag, ELEMENTWISE, lambda rb, x=x: {"sum": (rb.fromarray(x).sum(), want_sum(x)),
                                                    "strided": (rb.fromarray(x)[::3].sum(), want_sum(x[::3])),
                                                    "reversed": (rb.fromarray(x)[::-1].sum(), want_sum(x[::-1])),
                                                    "module": (rb.sum(rb.fromarray(x)), want_sum(x))})
        m = full_range(rows * 37, dt, 11).reshape(rows, 37)
        add("axis_sum_%s" % tag, T.AXIS_SPLIT, lambda rb, m=m: {
            "ax0": (rb.fromarray(m).sum(axis=0), want_sum(m, 0)), "ax1": (rb.fromarray(m).sum(axis=1), want_sum(m, 1)),
            "T": (rb.fromarray(m).T.sum(axis=0), want_sum(m.T, 0)),
            "keep": (rb.fromarray(m).sum(axis=0, keepdims=True), want_sum(m, 0).reshape(1, -1))})
        mk = onp.random.default_rng(12).random(n1) < 0.6
        add("masked_sum_%s" % tag, ELEMENTWISE, lambda rb, x=x, mk=mk: {
            "sum": (rb.fromarray(x)[rb.fromarray(mk)].sum(), want_sum(x[mk]))})
        p = odd_factors(4099 if not big else 1 << 20, dt, 13)
        pm = p[:4096].reshape(-1, 32)
        add("prod_%s" % tag, (ELEMENTWISE, INTERP + " form=axis_reduce"), lambda rb, p=p, pm=pm: {
            "prod": (rb.fromarray(p).prod(), want_prod(p)),
            "axis": (rb.fromarray(pm).prod(axis=0), onp.array([want_prod(c) for c in pm.T], dtype=p.dtype))})
        if dt != onp.bool_:
            add("minmax_pos_%s" % tag, (ELEMENTWISE,) + T.AXIS_SPLIT, lambda rb, dt=dt: _minmax_positions(rb, npos, dt))
            md = mean_data((n1,), dt, 14)
            mm = mean_data((rows, 37), dt, 15)
            add("mean_%s" % tag, (ELEMENTWISE,) + T.AXIS_SPLIT, lambda rb, md=md, mm=mm: {
                "mean": (onp.float64(rb.fromarray(md).mean()), want_mean(md)),
                "nanmean": (onp.float64(rb.nanmean(rb.fromarray(md))), want_mean(md)),
                "module": (onp.float64(rb.mean(rb.fromarray(md))), want_mean(md)),
                "ax0": (rb.fromarray(mm).mean(axis=0), want_mean(mm, 0)), "ax1": (rb.fromarray(mm).mean(axis=1), want_mean(mm, 1))})
        else:
            b = mean_data((n1,), dt, 14)
            add("mean_bool", ELEMENTWISE, lambda rb, b=b: {"mean": (onp.float64(rb.fromarray(b).mean()), want_mean(b)),
                                                     "ones": (onp.float64(rb.fromarray(onp.ones(300, bool)).mean()), onp.float64(1.0))})
        if dt != onp.bool_:
            add("truth_%s" % tag, INTERP, lambda rb, dt=dt: _truth_cases(rb, npos, dt))
        s = full_range(nscan, dt, 16)
        s2 = full_range(rows * 37, dt, 17).reshape(rows, 37)
        add("cumsum_%s" % tag, (lambda pl, big=big: pl.startswith("kernel=scan form=lookback") and (not big or int(pl.split("tiles=")[1]) > 2400),
                                "kernel=scan form=columns"),
            lambda rb, s=s, s2=s2: {"1d": (rb.cumsum(rb.fromarray(s)), want_cumsum(s, 0)),
                                    "ax0": (rb.cumsum(rb.fromarray(s2), axis=0), want_cumsum(s2, 0)),
                                    "ax1": (rb.cumsum(rb.fromarray(s2), axis=1), want_cumsum(s2, 1))})
    for dt in (onp.float64, onp.float32):
        add("truth_%s" % onp.dtype(dt).name, INTERP, lambda rb, dt=dt: _truth_cases(rb, npos, dt))
    add("truth_bool", INTERP, lambda rb: _truth_cases(rb, npos, onp.bool_))
    add("truth_forms", (INTERP + " form=elementwise", INTERP + " form=axis_as_1d", INTERP + " form=axis_reduce", "kernel=reduce_partials"),
        lambda rb: _truth_forms(rb, rows))
    add("sum_dtype", (ELEMENTWISE,) + T.AXIS_SPLIT, _sum_dtype)
    for dt in (onp.int64, onp.int32, onp.uint32):
        sc = odd_factors(nscan // 4, dt, 18)
        sm = full_range(nscan // 4, dt, 19)
        f = {"min": onp.minimum, "max": onp.maximum}
        add("scumulative_%s" % onp.dtype(dt).name, "kernel=scan form=lookback", lambda rb, sc=sc, sm=sm, f=f: dict(
            [("scum%s" % k, (rb.scumulative(g, g, rb.fromarray(sm)), getattr(onp, k + "imum").accumulate(sm.astype(onp.int64)))) for k, g in f.items()]
            + [("scumprod", (rb.scumulative(lambda a, b: a * b, lambda a, b: a * b, rb.fromarray(sc)), want_cumprod(sc)))]))
    for gname, shape, dim, G, gform in T.GROUP_CASES:
        for dt in (onp.int64, onp.int32, onp.uint32, onp.int8, onp.bool_):
            add("group_%s_%s" % (gname, onp.dtype(dt).name), gform, lambda rb, shape=shape, dim=dim, G=G, dt=dt: _group(rb, shape, dim, G, dt))
    return cases


def _minmax_positions(rb, n, dt):
    out = {}
    for which in ("min", "max"):
        for p in positions(n):
            x = minmax_data(n, dt, p, which, p)
            out["%s_%d" % (which, p)] = (getattr(rb.fromarray(x), which)(), getattr(x, which)())
        x = minmax_data(n, dt, 1, which, n // 3)
        out["%s_module" % which] = (getattr(rb, which)(rb.fromarray(x)), getattr(x, which)())
        out["%s_reversed" % which] = (getattr(rb.fromarray(x)[::-1], which)(), getattr(x, which)())
        mk = onp.ones(n, dtype=bool)
        mk[n // 3] = False  # the extreme is masked out
        out["%s_masked" % which] = (getattr(rb.fromarray(x)[rb.fromarray(mk)], which)(), getattr(x[mk], which)())
        m = minmax_data(4099 * 37, dt, 2, which, 4099 * 18 + 5).reshape(4099, 37)
        out["%s_ax0" % which] = (getattr(rb.fromarray(m), which)(axis=0), getattr(m, which)(axis=0))
        out["%s_ax1" % which] = (getattr(rb.fromarray(m), which)(axis=1), getattr(m, which)(axis=1))
        if dt in (onp.int64, onp.uint32) and not (dt == onp.uint32 and which == "max"):
            w = wide_minmax(n, which, dt, 3)
            out["%s_wide" % which] = (getattr(rb.fromarray(w), which)(), getattr(w, which)())
    return out


def _truth_cases(rb, n, dt):
    """any: cancelling pairs, one nonzero at each position class, -0.0 alone; all: wrapping / underflowing / NaN-making
    products, one zero at each position class."""
    out = {}
    isf = onp.dtype(dt).kind == "f"

    def both(label, x):
        A = rb.fromarray(x)
        out[label + "_any"] = (A.any(), onp.bool_(any(truth(x))))
        out[label + "_all"] = (A.all(), onp.bool_(all(truth(x))))

    if isf:
        tiny, huge = (1e-200, 1e308) if dt == onp.float64 else (1e-30, 3e38)
        both("cancel", onp.array([0.5, -0.5] * 50 + [0.0], dtype=dt))
        both("tiny", onp.full(4099, tiny, dtype=dt))
        both("nan0", onp.array([onp.nan, 0.0], dtype=dt))
        both("nan", onp.concatenate([onp.ones(4099), [onp.nan]]).astype(dt))
        both("huge0", onp.array([huge, -huge, 0.0], dtype=dt))
        both("negzero", onp.full(4099, -0.0, dtype=dt))
    elif dt != onp.bool_:
        both("cancel", any_cancel(n, dt))
        both("twos", all_wrap(n, dt))
        both("full2", onp.full(64, 2, dtype=dt))
        both("extreme", onp.array([onp.iinfo(dt).min, onp.iinfo(dt).max, 1], dtype=dt))
    for p in positions(n):
        z = onp.zeros(n, dtype=dt)
        z[p] = 1 if not isf else -0.25
        out["one_%d" % p] = (rb.fromarray(z).any(), onp.bool_(True))
        o = onp.ones(n, dtype=dt)
        if dt != onp.bool_:
            o[:] = 3 if not isf else 1e-200 if dt == onp.float64 else 1e-30
        o[p] = 0
        out["zero_%d" % p] = (rb.fromarray(o).all(), onp.bool_(False))
    o = onp.ones(n, dtype=dt)
    out["ones_all"] = (rb.fromarray(o).all(), onp.bool_(True))
    out["zeros_any"] = (rb.fromarray(onp.zeros(n, dtype=dt)).any(), onp.bool_(False))
    if dt != onp.bool_:
        x = any_cancel(n, dt) if not isf else onp.where(onp.arange(n) % 2 == 0, 0.5, -0.5).astype(dt)
        mk = onp.zeros(n, dtype=bool)
        mk[[1, n - 2]] = True
        out["masked_any"] = (rb.fromarray(x)[rb.fromarray(mk)].any(), onp.bool_(any(truth(x[mk]))))
        out["module_any"] = (rb.any(rb.fromarray(x)), onp.bool_(any(truth(x))))
        y = all_wrap(n, dt) if not isf else onp.full(n, 1e-200 if dt == onp.float64 else 1e-30, dtype=dt)
        out["masked_all"] = (rb.fromarray(y)[rb.fromarray(~mk)].all(), onp.bool_(all(truth(y[~mk]))))
        out["module_all"] = (rb.all(rb.fromarray(y)), onp.bool_(all(truth(y))))
    return out


def _truth_forms(rb, rows):
    """all / any along axes on data whose products wrap and sums cancel: the interpreter's axis forms and the fold of
    split partials."""
    out = {}
    r = onp.random.default_rng(30)
    for dt in (onp.int64, onp.int8, onp.uint8, onp.float64):
        isf = dt == onp.float64
        m = onp.ones((rows, 37), dtype=dt) * (2 if not isf else 1e-200)
        m[r.integers(0, rows, 40), r.integers(0, 37, 40)] = 0
        c = onp.zeros((rows, 37), dtype=onp.int64)
        c[0], c[-1] = 1, (-1 if dt != onp.uint8 else 255)
        c[rows // 2, 3], c[rows // 2 + 1, 3] = 2, (-2 if dt != onp.uint8 else 254)
        c = c.astype(dt)
        for ax in (0, 1):
            tag = "%s_ax%d" % (onp.dtype(dt).name, ax)
            out["all_" + tag] = (rb.fromarray(m).all(axis=ax), onp.array(truth(m), dtype=bool).reshape(m.shape).all(axis=ax))
            out["any_" + tag] = (rb.fromarray(c).any(axis=ax), onp.array(truth(c), dtype=bool).reshape(c.shape).any(axis=ax))
        out["allT_%s" % onp.dtype(dt).name] = (rb.fromarray(m).T.all(axis=0), onp.array(truth(m), dtype=bool).reshape(m.shape).all(axis=1))
        out["anykeep_%s" % onp.dtype(dt).name] = (rb.fromarray(c).any(axis=0, keepdims=True),
                                                  onp.array(truth(c), dtype=bool).reshape(c.shape).any(axis=0, keepdims=True))
        big = onp.ones((3001, 4096), dtype=dt) * (2 if not isf else 1e-200)
        big[1500, 4000] = 0
        out["all_cols_%s" % onp.dtype(dt).name] = ((rb.fromarray(big) + 0 * rb.sin(rb.fromarray(big))).all(axis=0),
                                                   onp.array([j != 4000 for j in range(4096)]))
    return out


def _sum_dtype(rb):
    """sum / prod(dtype=D): each element converted to D first (NumPy's rule), global and axis forms.  float64 data are
    chosen so that every float64 partial is exact: m * 2^40 + low bits that the conversion rounds away."""
    r = onp.random.default_rng(40)
    out = {}
    x = (r.integers(1 << 19, 1 << 20, size=(4099, 5), dtype=onp.int64) * r.choice([-1, 1], size=(4099, 5))) << 40
    x = x | r.integers(0, 1 << 6, size=x.shape, dtype=onp.int64)
    conv = [[Fraction(float(onp.float64(v))) for v in row] for row in x.tolist()]
    tot = sum(sum(row) for row in conv)
    assert float(tot) == tot
    out["sum_f64"] = (onp.float64(rb.fromarray(x).sum(dtype=onp.float64)), onp.float64(float(tot)))
    out["sum_f64_ax0"] = (rb.fromarray(x).sum(axis=0, dtype=onp.float64), onp.array([float(sum(c)) for c in zip(*conv)]))
    out["sum_f64_full"] = (onp.float64(rb.fromarray(onp.full((3, 5), 2 ** 60 + 1)).sum(dtype=onp.float64)), onp.float64(15 * 2.0 ** 60))
    p = onp.ones(300, dtype=onp.int64)
    p[[3, 100, 299]] = 1 << 40
    p[[5, 7]] = 3
    out["prod_f64"] = (onp.float64(rb.fromarray(p).prod(dtype=onp.float64)), onp.float64(float(9 * (1 << 120))))
    out["prod_f64_pair"] = (onp.float64(rb.fromarray(onp.array([2 ** 40, 2 ** 40])).prod(dtype=onp.float64)), onp.float64(2.0 ** 80))
    for dt in (onp.int8, onp.uint8, onp.int32, onp.uint32, onp.bool_):
        y = full_range(10007, dt, 41)
        out["sum_i64_%s" % onp.dtype(dt).name] = (rb.fromarray(y).sum(dtype=onp.int64), onp.int64(exact_total(y)))
        out["sum_f64_%s" % onp.dtype(dt).name] = (onp.float64(rb.fromarray(y).sum(dtype=onp.float64)), onp.float64(exact_total(y)))
    return out


def _group(rb, shape, dim, G, dt):
    """groupby sum / prod (source dtype, wrapping), min / max, count and mean (float64 sum / count) against the models."""
    r = onp.random.default_rng(G + 50)
    labels = onp.random.default_rng(G).integers(0, G, shape[dim])
    members = [onp.flatnonzero(labels == g) for g in range(G)]
    n = int(onp.prod(shape))
    out = {}
    x = full_range(n, dt, G + 51).reshape(shape)
    xi = onp.moveaxis(x, dim, -1)

    def per_group(fn, src, odt):
        res = onp.stack([onp.array([fn(row[mem]) for row in src.reshape(-1, src.shape[-1])], dtype=object).reshape(src.shape[:-1])
                         for mem in members], axis=-1)
        return onp.moveaxis(res.astype(odt), -1, dim)

    gb = rb.fromarray(x).groupby(dim, labels, G)
    out["sum"] = (gb.sum(), per_group(lambda v: wrap(exact_total(v), dt), xi, dt))
    if dt != onp.bool_:
        lo, hi = (int(onp.iinfo(dt).min), int(onp.iinfo(dt).max))
        out["min"] = (gb.min(), per_group(lambda v: int(v.min()) if v.size else hi, xi, dt))
        out["max"] = (gb.max(), per_group(lambda v: int(v.max()) if v.size else lo, xi, dt))
    out["count"] = (gb.count(), per_group(lambda v: v.size, xi, onp.int64))
    f = odd_factors(n, dt, G + 52).reshape(shape)
    out["prod"] = (rb.fromarray(f).groupby(dim, labels, G).prod(), per_group(lambda v: want_prod(v), onp.moveaxis(f, dim, -1), dt))
    md = mean_data(shape, dt, G + 53)
    with onp.errstate(all="ignore"):
        out["mean"] = (rb.fromarray(md).groupby(dim, labels, G).mean(),
                       per_group(lambda v: float(Fraction(exact_total(v), v.size)) if v.size else onp.nan, onp.moveaxis(md, dim, -1), onp.float64))
    return out


def _value(v):
    import ramba_b200 as rb

    return onp.asarray(v.asarray() if isinstance(v, rb.ndarray) else v)


def evaluate(size, only=None):
    """Run every case: ({case: {label: n_bad}}, {case: [plans of its op lists and kernel calls]})."""
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
            vals = {k: (_value(g), onp.asarray(w)) for k, (g, w) in got.items()}
            rb.sync()
        finally:
            be.run = run
            del RT.cumulative, RT.reduce_partials, RT.group_reduce
        res = {}
        for label, (g, w) in vals.items():
            try:
                res[label] = same_bits(g, w)
            except AssertionError as e:  # dtype or shape differs
                res[label] = "%s: %s" % (label, e)
        results[name] = res
        print("case %s done" % name, file=sys.stderr, flush=True)
        plans[name] = seen
        del got, vals
    return results, plans


def check(results, plans, size, forms=True):
    forms = {name: (form if forms else None) for name, form, _ in _cases(size)}
    for name, res in results.items():
        for label, v in res.items():
            assert v == 0, (name, label, v)
        if forms[name] is not None:
            for f in forms[name] if isinstance(forms[name], tuple) else (forms[name],):
                hit = f if callable(f) else (lambda p, f=f: p.startswith(f))
                assert any(hit(p) for p in plans[name]), (name, f, plans[name])
        if name.startswith("truth"):  # bool partials stay off the streaming kernels
            assert not any(p.startswith(("kernel=stream", "kernel=mapred")) for p in plans[name]), (name, plans[name])
    reached = sorted({" ".join(p.split()[:2]) for ps in plans.values() for p in ps})
    return reached


# every plan form the whole set of cases must reach
FORMS = ("kernel=general_interpreter form=elementwise", "kernel=general_interpreter form=axis_as_1d",
         "kernel=general_interpreter form=axis_reduce", "kernel=reduce_partials", "kernel=scan form=lookback",
         "kernel=scan form=columns", "kernel=group form=row", "kernel=group form=column", "kernel=group form=general")


def test_oracle_cases(oracle_engine):
    results, plans = evaluate("small")
    reached = check(results, plans, "small")
    for f in FORMS:
        assert any(r.startswith(f) for r in reached), (f, reached)
    print("forms reached (oracle):", json.dumps(reached))


# ---- several ranks ------------------------------------------------------------------------------------------------------
def world_sources():
    """(name, array, [(op, axis)]): every rank builds the same values.  Positions of the extremes and of the single
    nonzero / zero are chosen in the worker from the distribution (both sides of every rank boundary)."""
    out = []
    for dt in (onp.int64, onp.int32, onp.uint32, onp.int8, onp.uint8, onp.bool_):
        tag = onp.dtype(dt).name
        out.append(("v_%s" % tag, full_range(40009, dt, 60), [("sum", None), ("cumsum", 0), ("min", None), ("max", None)]))
        out.append(("m_%s" % tag, full_range(3001 * 7, dt, 61).reshape(3001, 7), [("sum", 0), ("sum", 1), ("sum", None), ("cumsum", 0), ("cumsum", 1)]))
        out.append(("p_%s" % tag, odd_factors(4001, dt, 62), [("prod", None)]))
        if dt != onp.bool_:
            out.append(("mean_%s" % tag, mean_data((4001,), dt, 63), [("mean", None)]))
            out.append(("mean2_%s" % tag, mean_data((1001, 5), dt, 64), [("mean", 0), ("mean", 1)]))
            out.append(("cancel_%s" % tag, any_cancel(4001, dt), [("any", None), ("all", None)]))
            out.append(("twos_%s" % tag, all_wrap(4001, dt), [("any", None), ("all", None)]))
    for dt in (onp.float64, onp.float32):
        out.append(("fcancel_%s" % onp.dtype(dt).name, onp.where(onp.arange(4001) % 2 == 0, 0.5, -0.5).astype(dt), [("any", None), ("all", None)]))
        out.append(("ftiny_%s" % onp.dtype(dt).name, onp.full(4001, 1e-200 if dt == onp.float64 else 1e-30, dtype=dt), [("all", None)]))
    return out


def _expected_world(x, op, axis):
    if op == "sum":
        return want_sum(x, axis)
    if op == "prod":
        return want_prod(x)
    if op == "cumsum":
        return want_cumsum(x, axis)
    if op == "mean":
        return want_mean(x, axis)
    if op in ("any", "all"):
        return onp.bool_(getattr(builtins_mod, op)(truth(x)))
    return getattr(x, op)(axis=axis)


def _run_world(world, out):
    port = T._free_port()
    procs = []
    for r in range(world):
        env = dict(os.environ)
        env.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r), "MASTER_ADDR": "127.0.0.1",
                    "MASTER_PORT": str(port), "OMP_NUM_THREADS": "1"})
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_intred_worker.py"), out], env=env,
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


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_worlds_match_the_exact_models(tmp_path, world):
    res = _run_world(world, str(tmp_path / "w.npz"))
    split = 0
    for name, x, ops in world_sources():
        blocks = res[name + ".blocks"]
        split += int((blocks[:, x.ndim:] > 0).all(axis=1).sum() > 1)
        for op, axis in ops:
            key = "%s.%s.%s" % (name, op, axis)
            assert_bits(res[key], _expected_world(x, op, axis), "W=%d %s" % (world, key))
    # the extremes, the single nonzero and the single zero on both sides of every rank boundary
    n = 0
    for key in res:
        if key.startswith("edge."):
            _, what, dtn, p = key.split(".")
            x = edge_data(what, onp.dtype(dtn).type, 4001, int(p))
            assert_bits(res[key], _expected_world(x, what.split("_")[0], None), "W=%d %s" % (world, key))
            n += 1
    assert split > 0 and n > 0


def edge_data(what, dt, n, p):
    """The arrays of the rank-boundary cases: min / max with the extreme at p, any with one nonzero at p, all with one
    zero at p."""
    op = what.split("_")[0]
    if op in ("min", "max"):
        return minmax_data(n, dt, 70, op, p)
    if op == "any":
        x = onp.zeros(n, dtype=dt)
        x[p] = 1
        return x
    x = onp.full(n, 2, dtype=dt) if dt != onp.bool_ else onp.ones(n, dtype=bool)
    x[p] = 0
    return x


# ---- GPU ----------------------------------------------------------------------------------------------------------------
SWITCHES, BARRED = T.SWITCHES, T.BARRED


def check_switched(switches, results, plans, size):
    if switches == "default":
        return check(results, plans, size)
    bar = BARRED[switches]
    for name, ps in plans.items():
        assert not any(bar(p) for p in ps), (switches, name, ps)
    return check(results, {k: [] for k in plans}, size, forms=False)


def _plans_worker(out_dir, switches):
    from ramba_b200.runtime import RT

    RT.reset()
    if switches != "gpu":
        import _oracle_backend

        _oracle_backend.install()
    elif os.environ.get("RB200_DRY_GPU_TESTS"):
        import conftest

        conftest._dry_gpu()
    with onp.errstate(all="ignore"):
        results, plans = evaluate("small" if switches != "gpu" else os.environ["RB200_INTRED_SIZE"])
    with open(os.path.join(out_dir, "out.json"), "w") as f:
        json.dump([results, plans], f)


def _run_switched(tmp_path, switches, backend, size="small"):
    code = "import sys; sys.path[:0] = [%r, %r]; import test_integer_reductions as t; t._plans_worker(%r, %r)" % (
        ROOT, HERE, str(tmp_path), "gpu" if backend == "gpu" else switches)
    env = dict(os.environ, RB200_INTRED_SIZE=size, **SWITCHES[switches])
    out = subprocess.run([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3000)
    assert out.returncode == 0, out.stdout[-3000:]
    with open(os.path.join(str(tmp_path), "out.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("switches", [s for s in SWITCHES if s != "default"])
def test_switched_kernels_on_the_oracle(tmp_path, switches):
    results, plans = _run_switched(tmp_path, switches, "oracle")
    check_switched(switches, results, plans, "small")


@pytest.mark.gpu
@pytest.mark.timeout(3600)
@pytest.mark.parametrize("switches", list(SWITCHES))
def test_integer_reductions_on_the_gpu(tmp_path, switches):
    size = "big" if switches == "default" else "small"
    results, plans = _run_switched(tmp_path, switches, "gpu", size)
    reached = check_switched(switches, results, plans, size)
    if switches == "default":
        for f in FORMS:
            assert any(r.startswith(f) for r in reached), (f, reached)
        print("forms reached (gpu):", json.dumps(reached))


@pytest.mark.gpu
@pytest.mark.timeout(1200)
def test_any_and_max_past_2_31_elements(gpu_engine):
    """any and max over 2^31 + 4099 uint8 elements, the only nonzero value or the maximum at 2^31 + k."""
    import torch

    import ramba_b200 as rb

    if os.environ.get("RB200_DRY_GPU_TESTS"):
        pytest.skip("2 GB arrays on the oracle")
    if torch.cuda.get_device_properties(0).total_memory < (24 << 30):
        pytest.skip("needs 24 GB")
    n = (1 << 31) + 4099
    A = rb.zeros(n, dtype=onp.uint8)
    for k in (3, 4097):
        A[(1 << 31) + k] = 200
        assert bool(A.any()) is True
        assert int(A.max()) == 200
        A[(1 << 31) + k] = 0
        assert bool(A.any()) is False
    B = (rb.arange(n) % 7).astype(onp.uint8)
    B[(1 << 31) + 5] = 255
    assert int(B.max()) == 255 and int(B.min()) == 0
    assert bool(B.all()) is False
    del A, B
