"""The shifted-view stencil / N-d float kernel (ramba_b200/csrc/rb200_tile.cu) against the oracle: same programs on
the oracle executor (CPU, always) and through the CUDA library (-m gpu), BIT-exact on arbitrary float data (both
sides do the same operations in the same order and classes, one rounding each).  Shapes cover the TMA path (row
strides that are multiples of 16 bytes), the cooperative cp.async path (odd row lengths, unaligned corners), ragged
tiles, 2-D and 3-D, float32 and float64, wide halos, several source arrays, in-place accumulation.

With np = NumPy each program computes its expected value with the engine's per-operation classes written out (Numba's
typing: float32 op float32 rounds in float32, float32 op a Python float is a float64 operation, the store converts), so
the oracle leg compares bit for bit too."""
import numpy as onp
import pytest


def _h(x):
    return x.asarray() if hasattr(x, "asarray") else onp.asarray(x)


def _f64(x):
    return onp.asarray(x).astype(onp.float64)


def _data(shape, dtype, seed):
    rng = onp.random.RandomState(seed)
    return (rng.rand(*shape) * 8 - 4).astype(dtype)


def lap3d(np, n0, n1, n2, dtype, seed=0):
    """7-point Laplacian written with slice views (BASELINE config 4's program, SURVEY §3.5)."""
    Uh = _data((n0, n1, n2), dtype, seed)
    U = Uh if np is onp else np.fromarray(Uh)
    V = np.zeros((n0, n1, n2), dtype=dtype)
    if np is onp:
        s = U[:-2, 1:-1, 1:-1] + U[2:, 1:-1, 1:-1] + U[1:-1, :-2, 1:-1] + U[1:-1, 2:, 1:-1] + U[1:-1, 1:-1, :-2] + U[1:-1, 1:-1, 2:]
        V[1:-1, 1:-1, 1:-1] = _f64(s) - 6.0 * _f64(U[1:-1, 1:-1, 1:-1])
        return [V]
    V[1:-1, 1:-1, 1:-1] = (U[:-2, 1:-1, 1:-1] + U[2:, 1:-1, 1:-1] + U[1:-1, :-2, 1:-1] + U[1:-1, 2:, 1:-1]
                           + U[1:-1, 1:-1, :-2] + U[1:-1, 1:-1, 2:] - 6.0 * U[1:-1, 1:-1, 1:-1])
    return [_h(V)]


def star2d(np, n, m, dtype, r, seed=1):
    """PRK-style star stencil of radius r with weights, accumulated into the output (README.md:271-299)."""
    Ah = _data((n, m), dtype, seed)
    A = _f64(Ah) if np is onp else np.fromarray(Ah)  # (every weighted term is a float64 operation)
    B = np.ones((n, m), dtype=dtype)
    acc = None
    for j in range(1, r + 1):
        w = 1.0 / (2.0 * j * r)
        t = (w * A[r:-r, r + j:m - r + j] - w * A[r:-r, r - j:m - r - j]
             + w * A[r + j:n - r + j, r:-r] - w * A[r - j:n - r - j, r:-r])
        if np is onp and j == r:
            # the last t is still named by a Python variable when B is updated, so the engine stores it (rounded to the
            # data's dtype); earlier t's and partial sums are never stored and keep their float64 values
            t = _f64(t.astype(dtype))
        acc = t if acc is None else acc + t
    if np is onp:
        acc = acc.astype(dtype)  # (acc is stored too)
    B[r:-r, r:-r] += acc
    return [_h(B)]


def box2d(np, n, m, dtype, seed=2):
    """3x3 box filter (corners included) times a second array read at the centre only."""
    Ah, Wh = _data((n, m), dtype, seed), _data((n, m), dtype, seed + 7)
    A, W = (Ah, Wh) if np is onp else (np.fromarray(Ah), np.fromarray(Wh))
    out = np.zeros((n, m), dtype=dtype)
    s = None
    for dy in (0, 1, 2):
        for dx in (0, 1, 2):
            v = A[dy:n - 2 + dy, dx:m - 2 + dx]
            s = v if s is None else s + v
    out[1:-1, 1:-1] = _f64(s * W[1:-1, 1:-1]) * 0.125 if np is onp else s * W[1:-1, 1:-1] * 0.125
    return [_h(out)]


def asym3d(np, n0, n1, n2, dtype, seed=3):
    """One-sided (upwind) differences: halos on one side only, two planes back in z."""
    Uh = _data((n0, n1, n2), dtype, seed)
    U = Uh if np is onp else np.fromarray(Uh)
    V = np.zeros((n0 - 2, n1 - 1, n2 - 3), dtype=dtype)
    if np is onp:
        V[:, :, :] = _f64(U[2:, 1:, 3:]) - 0.5 * _f64(U[1:-1, 1:, 3:]) - 0.25 * _f64(U[:-2, 1:, 3:]) + _f64(U[2:, :-1, 3:] * U[2:, 1:, :-3])
        return [V]
    V[:, :, :] = U[2:, 1:, 3:] - 0.5 * U[1:-1, 1:, 3:] - 0.25 * U[:-2, 1:, 3:] + U[2:, :-1, 3:] * U[2:, 1:, :-3]
    return [_h(V)]


def elementwise_nd(np, shape, dtype, seed=4):
    """No shifted views at all: N-d float arithmetic over strided / broadcast / transposed operands."""
    Ah, Bh = _data(shape, dtype, seed), _data(shape, dtype, seed + 1)
    A, B = (Ah, Bh) if np is onp else (np.fromarray(Ah), np.fromarray(Bh))
    row = A[0] * 2.0
    sl = tuple(slice(1, None, 2) for _ in shape)
    if np is onp:
        dt = Ah.dtype
        return [(_f64(A[sl] * B[sl]) - 0.5 * _f64(A[sl])).astype(dt), (_f64(A + row) * 0.5).astype(dt),
                (abs(_f64(A.T) - 1.0) + _f64(B.T * B.T)).astype(dt), (_f64(onp.minimum(A[sl], B[sl])) - onp.maximum(_f64(A[sl]), 0.25)).astype(dt)]
    return [_h(A[sl] * B[sl] - 0.5 * A[sl]), _h((A + row) * 0.5), _h(abs(A.T - 1.0) + B.T * B.T), _h(np.minimum(A[sl], B[sl]) - np.maximum(A[sl], 0.25))]


CASES = [
    ("lap3d_tma_f32", lambda np: lap3d(np, 20, 36, 132, onp.float32)),        # rows of 132 floats: 16-byte multiples -> TMA
    ("lap3d_tma_f64", lambda np: lap3d(np, 12, 40, 130, onp.float64)),
    ("lap3d_odd_f32", lambda np: lap3d(np, 9, 35, 131, onp.float32)),         # odd rows -> cooperative loader
    ("lap3d_odd_f64", lambda np: lap3d(np, 7, 21, 67, onp.float64)),
    ("lap3d_ragged_f32", lambda np: lap3d(np, 40, 50, 300, onp.float32)),     # several tiles in x and y, ragged edges
    ("lap3d_narrow_f32", lambda np: lap3d(np, 33, 70, 24, onp.float32)),      # TX = 32
    ("lap3d_mid_f32", lambda np: lap3d(np, 18, 90, 60, onp.float32)),         # TX = 64
    ("star2d_r1_f32", lambda np: star2d(np, 200, 260, onp.float32, 1)),
    ("star2d_r2_f32", lambda np: star2d(np, 129, 257, onp.float32, 2)),
    ("star2d_r4_f64", lambda np: star2d(np, 150, 272, onp.float64, 4)),
    ("box2d_f32", lambda np: box2d(np, 100, 260, onp.float32)),
    ("box2d_f64", lambda np: box2d(np, 77, 199, onp.float64)),
    ("asym3d_f32", lambda np: asym3d(np, 11, 30, 140, onp.float32)),
    ("asym3d_f64", lambda np: asym3d(np, 8, 19, 95, onp.float64)),
    ("elementwise_2d_f32", lambda np: elementwise_nd(np, (130, 270), onp.float32)),
    ("elementwise_3d_f64", lambda np: elementwise_nd(np, (11, 50, 70), onp.float64)),
]


def _exact(got, exp, name):
    assert len(got) == len(exp)
    for i, (g, e) in enumerate(zip(got, exp)):
        assert g.shape == e.shape and g.dtype == e.dtype, "%s[%d]: %s %s vs %s %s" % (name, i, g.shape, g.dtype, e.shape, e.dtype)
        assert onp.array_equal(g, e), "%s[%d]: %d elements differ, max |d| = %g" % (
            name, i, int((g != e).sum()), float(onp.max(onp.abs(g.astype(onp.float64) - e.astype(onp.float64)))))


@pytest.mark.parametrize("name,prog", CASES, ids=[c[0] for c in CASES])
def test_stencil_oracle_vs_numpy(oracle_engine, name, prog):
    """Host logic + oracle: the op list the fuser builds means what the program's NumPy restatement computes with the
    engine's per-operation classes, bit for bit."""
    import ramba_b200 as rb

    _exact(prog(rb), prog(onp), name)


@pytest.mark.gpu
@pytest.mark.parametrize("name,prog", CASES, ids=[c[0] for c in CASES])
def test_stencil_cuda_matches_oracle(gpu_engine, name, prog):
    import _oracle_backend
    import ramba_b200 as rb
    from ramba_b200 import _cabi, ramba
    from ramba_b200.runtime import RT

    before = _cabi.launch_count()
    got = prog(rb)
    assert RT.is_cuda and _cabi.launch_count() > before, "the CUDA library did not run"
    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()
    _oracle_backend.install()
    try:
        exp = prog(rb)
    finally:
        ramba.deferred_op.ramba_deferred_ops = None
        RT.reset()
    _exact(got, exp, name)
