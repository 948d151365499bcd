"""The fuser memoises lowered op lists on the structure of the pending statements (ramba_b200/ramba.py::_lower; the
reference's counterpart is Numba's compile cache keyed by the generated source, ramba/ramba.py:8247-8265).  A wrong
key would silently run the wrong op list, so: every program is run twice in one process with the memo checked against
a fresh lowering, and programs that differ ONLY in what the key must capture are run back to back."""
import numpy as onp
import pytest

import _random_programs


@pytest.fixture
def verified_memo(oracle_engine, monkeypatch):
    from ramba_b200 import ramba

    monkeypatch.setattr(ramba, "_VERIFY_LOWER_CACHE", True)
    return ramba


def test_hits_are_identical_to_fresh_lowerings(verified_memo):
    import ramba_b200 as rb

    verified_memo._lower_cache.clear()
    for f in _random_programs.CASES[:24]:
        first = f(rb)
        n = len(verified_memo._lower_cache)
        second = f(rb)  # same structure: served by the memo, verified against a fresh lowering
        assert len(verified_memo._lower_cache) == n, f.__name__
        for a, b in zip(first, second):
            assert onp.array_equal(onp.asarray(a), onp.asarray(b), equal_nan=True), f.__name__


def test_repeated_step_skips_lowering(oracle_engine, monkeypatch):
    import ramba_b200 as rb
    from ramba_b200 import ramba

    calls = []
    orig = ramba.deferred_op._lower_uncached

    def counted(self, *a, **k):
        calls.append(1)
        return orig(self, *a, **k)

    monkeypatch.setattr(ramba.deferred_op, "_lower_uncached", counted)
    monkeypatch.setattr(ramba, "_VERIFY_LOWER_CACHE", False)  # (the verification mode lowers every time by design)
    ramba._lower_cache.clear()
    A = rb.arange(1000) / 1000.0
    rb.sync()
    for it in range(4):
        calls.clear()
        B = rb.sin(A)
        C = rb.cos(A)
        D = B * B + C ** 2
        rb.sync()
        assert len(calls) == (1 if it == 0 else 0)
    assert onp.allclose(D.asarray(), 1.0)


@pytest.mark.parametrize("pair", [
    (0.0, -0.0),            # equal and equal-hashing as Python floats, different bits
    (2, 2.0),               # int64 vs float64 scalar class
    (True, 1),              # bool vs int
    (onp.float32(0.1), 0.1),  # float32 scalar keeps a float32 expression in float32
    (3.0, 3.5),
], ids=["signed_zero", "int_float", "bool_int", "f32_f64", "value"])
def test_scalars_are_part_of_the_key(verified_memo, pair):
    import ramba_b200 as rb

    x = onp.linspace(-2, 2, 41).astype(onp.float32)

    def run(s):
        a = rb.fromarray(x)
        with onp.errstate(divide="ignore"):
            return (a * s).asarray() if isinstance(s, bool) else (a * s + 1 / (a + s)).asarray()

    cold = []
    for s in pair:  # every program lowered from scratch
        verified_memo._lower_cache.clear()
        cold.append(run(s))
    verified_memo._lower_cache.clear()
    for s, c in list(zip(pair, cold)) * 2:  # back to back through the memo
        got = run(s)
        assert got.dtype == c.dtype, s
        assert onp.array_equal(got, c, equal_nan=True), s
    if pair == (0.0, -0.0):
        a = rb.fromarray(onp.ones(4))
        for z in (0.0, -0.0, 0.0, -0.0):  # 1 / (+-0 * a): the sign of the scalar decides the sign of the infinity
            with onp.errstate(divide="ignore"):
                assert onp.array_equal((1.0 / (a * z)).asarray(), 1.0 / (onp.ones(4) * z)), z


def test_aliasing_and_liveness_are_part_of_the_key(verified_memo):
    import ramba_b200 as rb

    x = onp.arange(64, dtype=onp.float64)
    # same operators, different operand identity: a+a vs a+b
    for _ in range(2):
        a, b = rb.fromarray(x), rb.fromarray(x * 2)
        assert onp.array_equal((a + a).asarray(), x + x)
        assert onp.array_equal((a + b).asarray(), x + x * 2)
    # same statements, the temporary alive (stored) or dead (register only)
    for _ in range(2):
        a = rb.fromarray(x)
        t = a * 2.0
        u = t + 1.0
        rb.sync()
        assert onp.array_equal(t.asarray(), x * 2) and onp.array_equal(u.asarray(), x * 2 + 1)
        a = rb.fromarray(x)
        u = a * 2.0 + 1.0
        assert onp.array_equal(u.asarray(), x * 2 + 1)
    # two views of one array vs views of two arrays (alias analysis of dead-store elimination)
    for _ in range(2):
        a = rb.fromarray(x.copy())
        a[1:] = a[:-1] + 1.0
        e = x.copy()
        e[1:] = e[:-1] + 1.0
        assert onp.array_equal(a.asarray(), e)
        a, c = rb.fromarray(x.copy()), rb.fromarray(x.copy())
        a[1:] = c[:-1] + 1.0
        assert onp.array_equal(a.asarray(), e)


def test_dtypes_are_part_of_the_key(verified_memo):
    import ramba_b200 as rb

    for dt in (onp.float64, onp.float32, onp.int64, onp.int32, onp.float64):
        x = onp.arange(32).astype(dt)
        got = (rb.fromarray(x) * 3 + 1).asarray()
        exp = x * 3 + 1
        assert got.dtype == exp.dtype and onp.array_equal(got, exp)


# ---- the flush memo (flush.py::run_deferred_ops): every flush is planned once per key into a script, and every flush
# runs its key's script
@pytest.fixture
def verified_plans(oracle_engine, monkeypatch):
    from ramba_b200 import flush

    monkeypatch.setattr(flush, "_VERIFY_PLAN_CACHE", True)
    flush._plan_cache.clear()
    return flush


def test_repeated_flush_runs_its_script_without_planning_again(verified_plans, monkeypatch):
    import ramba_b200 as rb

    planned = []
    orig = verified_plans._plan

    def counted(*a, **k):
        planned.append(1)
        return orig(*a, **k)

    monkeypatch.setattr(verified_plans, "_plan", counted)
    x = onp.arange(5000, dtype=onp.float64) / 7.0
    A = rb.fromarray(x)
    U = rb.fromarray(onp.arange(20 * 30 * 40, dtype=onp.float32).reshape(20, 30, 40) % 17)
    V = rb.zeros((20, 30, 40), dtype=onp.float32)
    rb.sync()

    def step():
        B = rb.sin(A)
        D = B * B + rb.cos(A) ** 2
        rb.sync()
        V[1:-1, 1:-1, 1:-1] = (U[:-2, 1:-1, 1:-1] + U[2:, 1:-1, 1:-1] + U[1:-1, :-2, 1:-1] + U[1:-1, 2:, 1:-1]
                               + U[1:-1, 1:-1, :-2] + U[1:-1, 1:-1, 2:] - 6.0 * U[1:-1, 1:-1, 1:-1])
        rb.sync()
        s = float((A * 2.0 + 1.0).sum())  # a global reduction: the reduction output pointer is patched as well
        return D, s

    monkeypatch.setattr(verified_plans, "_VERIFY_PLAN_CACHE", False)  # (the verification mode plans every hit again)
    for it in range(4):
        planned.clear()
        D, s = step()
        assert len(planned) == (3 if it == 0 else 0), (it, len(planned))
        assert onp.allclose(D.asarray(), 1.0)
        assert s == float((x * 2.0 + 1.0).sum())
    # verified: planning each of the three flushes again must give its memoised script
    monkeypatch.setattr(verified_plans, "_VERIFY_PLAN_CACHE", True)
    planned.clear()
    D, s = step()
    assert len(planned) == 3
    assert onp.allclose(D.asarray(), 1.0)
    assert s == float((x * 2.0 + 1.0).sum())
    u = onp.asarray(U.asarray())
    e = onp.zeros_like(u)
    e[1:-1, 1:-1, 1:-1] = (u[:-2, 1:-1, 1:-1] + u[2:, 1:-1, 1:-1] + u[1:-1, :-2, 1:-1] + u[1:-1, 2:, 1:-1] + u[1:-1, 1:-1, :-2]
                          + u[1:-1, 1:-1, 2:] - 6.0 * u[1:-1, 1:-1, 1:-1])
    assert onp.array_equal(V.asarray(), e)


def test_plan_memo_executes_once_and_follows_the_buffers(verified_plans, monkeypatch):
    import ramba_b200 as rb

    for verify in (False, True):  # hits replayed, then hits planned again and checked against the memoised scripts
        monkeypatch.setattr(verified_plans, "_VERIFY_PLAN_CACHE", verify)
        a = rb.fromarray(onp.zeros(1000))
        for it in range(5):
            a += 1.0  # in place: a flush executed twice (or against a stale buffer) would show
            rb.sync()
        assert onp.array_equal(a.asarray(), onp.full(1000, 5.0))
        outs = []
        for it in range(4):  # fresh result buffers every iteration, all alive at the end
            outs.append(a * float(2) + 1.0)
            rb.sync()
        for o in outs:
            assert onp.array_equal(o.asarray(), onp.full(1000, 11.0))
        # same op list over another layout: different script
        b = rb.fromarray(onp.ones((10, 100)))
        c = b[:, 1:] * 2.0 + 1.0
        d = b[:, :-1] * 2.0 + 1.0
        assert onp.array_equal(c.asarray(), onp.full((10, 99), 3.0)) and onp.array_equal(d.asarray(), onp.full((10, 99), 3.0))
