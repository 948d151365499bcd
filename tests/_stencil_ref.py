"""Data and comparison helpers of tests/test_stencil_semantics.py, shared with its gloo worker.

Expected values are never taken from the oracle, the op list or the fuser: every case writes its own NumPy expression
with explicit per-operation dtypes (float32 op float32 rounds in float32; float32 op a Python float or float64 is a
float64 operation; the store converts to the destination's dtype)."""
import numpy as onp

F32, F64 = onp.float32, onp.float64

# NaN, +-inf, -0.0, the smallest subnormal, a negative subnormal and a value whose double overflows float32
SPECIALS = {
    F32: [onp.nan, onp.inf, -onp.inf, -0.0, 1e-45, -3e-39, 3.0e38],
    F64: [onp.nan, onp.inf, -onp.inf, -0.0, 5e-324, -1e-310, 1.5e308],
}


def _edges(n, near):
    return sorted({i for c in near for i in (c - 1, c, c + 1) if 0 <= i < n} | {i for i in (n - 2, n - 1) if i >= 0})


def edge_data(shape, dtype, seed, specials=True):
    """uniform(-4, 4) data with NaN, +-inf, -0.0 and subnormals at the first and last column of a 128-wide tile and the
    columns of its halo (array columns 0-2, 127-130, 143-146: the box starts one column before the iteration box), the
    first and last row of a 16-row tile and the first and last plane of a 16-plane z-chunk"""
    r = onp.random.default_rng(seed)
    x = r.uniform(-4, 4, shape).astype(dtype)
    if not specials:
        return x
    sp = SPECIALS[dtype]
    nd = len(shape)
    axes = [_edges(shape[-1], (1, 128, 129, 144, 145))]
    if nd >= 2:
        axes.insert(0, _edges(shape[-2], (1, 16, 17)))
    if nd >= 3:
        axes.insert(0, _edges(shape[-3], (1, 16, 17)))
    k = 0
    for idx in onp.ndindex(*[len(a) for a in axes]):
        if sum(idx) % 3:
            continue
        x[tuple(a[i] for a, i in zip(axes, idx))] = sp[k % len(sp)]
        k += 1
    return x


def bits(x):
    x = onp.ascontiguousarray(onp.asarray(x))
    u = x.view(onp.uint64 if x.dtype.itemsize == 8 else onp.uint32).copy()
    u[onp.isnan(x)] = 1  # NaN as NaN, whatever its payload and sign
    return u


def mismatches(got, want, what):
    """[] when got and want hold the same bits (any NaN matches any NaN; zeros and infinities with their sign)"""
    out = []
    if len(got) != len(want):
        return ["%s: %d outputs, want %d" % (what, len(got), len(want))]
    for i, (g, w) in enumerate(zip(got, want)):
        g, w = onp.asarray(g), onp.asarray(w)
        if g.dtype != w.dtype or g.shape != w.shape:
            out.append("%s[%d]: %s %s, want %s %s" % (what, i, g.dtype, g.shape, w.dtype, w.shape))
            continue
        bad = bits(g) != bits(w)
        if bad.any():
            j = onp.argwhere(bad)[:3]
            out.append("%s[%d]: %d of %d differ, e.g. at %s got %r want %r" % (
                what, i, int(bad.sum()), bad.size, [tuple(int(v) for v in p) for p in j], [g[tuple(p)].item() for p in j],
                [w[tuple(p)].item() for p in j]))
    return out


def fma64(a, b, c):
    """a * b + c with ONE rounding (what a contracted multiply-add gives), float64, through exact rationals"""
    from fractions import Fraction

    a, b, c = onp.broadcast_arrays(onp.asarray(a, F64), onp.asarray(b, F64), onp.asarray(c, F64))
    out = onp.empty(a.shape, F64)
    for i in onp.ndindex(*a.shape):
        x, y, z = float(a[i]), float(b[i]), float(c[i])
        if not all(map(onp.isfinite, (x, y, z))):
            out[i] = x * y + z
        else:
            out[i] = float(Fraction(x) * Fraction(y) + Fraction(z))
    return out
