"""Host logic (API -> fuser -> lowering -> range binding) checked on CPU: op lists run through the
NumPy oracle instead of the CUDA kernels; results must equal plain NumPy running the same program
(the reference's run_both pattern, ramba/tests/test_distributed_array.py:255-259)."""
import numpy as onp
import pytest

import _programs


def _check(got, exp, name):
    assert len(got) == len(exp)
    for i, (g, e) in enumerate(zip(got, exp)):
        g, e = onp.asarray(g), onp.asarray(e)
        assert g.shape == e.shape, "%s[%d] shape %s vs %s" % (name, i, g.shape, e.shape)
        if e.dtype.kind == "f":
            assert onp.allclose(g, e, rtol=1e-13, atol=1e-15), "%s[%d]" % (name, i)
        else:
            assert onp.array_equal(g, e), "%s[%d]" % (name, i)


@pytest.mark.parametrize("prog", _programs.ALL, ids=lambda p: p.__name__)
def test_program_matches_numpy(oracle_engine, prog):
    import ramba_b200 as rb

    got = prog(rb)
    exp = prog(onp)
    _check(got, exp, prog.__name__)


def _captured_programs(monkeypatch):
    """Record the op list of every flush (the lowered Program objects)."""
    from ramba_b200 import ramba

    progs = []
    orig = ramba.run_deferred_ops

    def spy(views, prog, *args, **kwargs):
        progs.append(prog)
        return orig(views, prog, *args, **kwargs)

    monkeypatch.setattr(ramba, "run_deferred_ops", spy)
    return progs


def test_fusion_counts_like_the_reference(oracle_engine, monkeypatch):
    """TestFusion (ramba/tests/test_distributed_array.py:112-198): ten `a += 1` between two syncs are ONE
    fused op that reads and writes `a` once; ten `a[i:] += 1` cannot fuse (ten flushes); an expression with
    several temporaries materialises none of them."""
    import ramba_b200 as rb
    from ramba_b200 import _cabi

    progs = _captured_programs(monkeypatch)
    a = rb.zeros(1000, dtype=float)
    rb.sync()
    del progs[:]
    for _ in range(10):
        a += 1
    rb.sync()
    assert len(progs) == 1
    stores = [i for i in progs[0].insns if i["st_view"] != _cabi.NOSTORE]
    loads = [i for i in progs[0].insns for k in ("a", "b", "c") if i[k + "_kind"] == _cabi.K_VIEW]
    assert len(stores) == 1 and len(loads) == 1, "dead stores / repeated loads were not removed"
    assert onp.array_equal(a.asarray(), onp.full(1000, 10.0))

    del progs[:]
    for i in range(10):
        a[i:] += 1
    rb.sync()
    assert len(progs) == 10
    exp = onp.full(1000, 10.0)
    for i in range(10):
        exp[i:] += 1
    assert onp.array_equal(a.asarray(), exp)

    b = rb.ones(1000, dtype=float)
    rb.sync()
    del progs[:]
    b += (7 * b - 3) + (4 * b + 5 * b)
    assert b[0] == 14
    assert len(progs) == 1 and len({i["st_view"] for i in progs[0].insns if i["st_view"] != _cabi.NOSTORE}) == 1


def test_dead_store_elimination_respects_masks_and_aliases(oracle_engine, monkeypatch):
    import ramba_b200 as rb

    b = rb.arange(200) * 1.0
    rb.sync()
    b[b > 100.0] = -1.0   # masked store: the elements it leaves alone must survive
    b += 1
    c = b[:-1] + 0        # reads b through another view
    b += 1
    rb.sync()
    e = onp.arange(200) * 1.0
    e[e > 100.0] = -1.0
    e += 1
    ce = e[:-1] + 0
    e += 1
    assert onp.array_equal(b.asarray(), e) and onp.array_equal(c.asarray(), ce)
    # unmasked store first, masked one after it: both must reach memory
    d = rb.zeros(150)
    rb.sync()
    d += 5
    d[d > 1.0] = 2.0
    d[rb.arange(150) % 2 == 0] = 7.0
    de = onp.zeros(150)
    de += 5
    de[de > 1.0] = 2.0
    de[onp.arange(150) % 2 == 0] = 7.0
    assert onp.array_equal(d.asarray(), de)


def test_a_failed_flush_poisons_what_it_was_to_write(oracle_engine, monkeypatch):
    """A fused op that fails takes its statements with it: the arrays they were to write must raise when read, not return
    whatever their shards hold (ADVICE r01); arrays of other ops are unaffected."""
    import ramba_b200 as rb
    from ramba_b200 import ramba

    a = rb.fromarray(onp.arange(300, dtype=onp.float64))
    other = rb.fromarray(onp.arange(50, dtype=onp.float64)) + 1.0
    assert onp.array_equal(other.asarray(), onp.arange(50) + 1.0)
    good = a * 2.0
    bad = a + 1.0
    orig = ramba.run_deferred_ops
    calls = []

    def failing(*args, **kw):
        calls.append(1)
        raise ramba.ProgramError("injected failure")

    monkeypatch.setattr(ramba, "run_deferred_ops", failing)
    with pytest.raises(ramba.ProgramError):
        rb.sync()
    monkeypatch.setattr(ramba, "run_deferred_ops", orig)
    assert calls
    for x in (good, bad):
        with pytest.raises(RuntimeError, match="fused op that failed"):
            x.asarray()
        with pytest.raises(RuntimeError, match="fused op that failed"):
            (x + 1.0).asarray()
    # the source and unrelated arrays are intact, and new work runs
    assert onp.array_equal(a.asarray(), onp.arange(300))
    assert onp.array_equal((a * 3.0).asarray(), onp.arange(300) * 3.0)
    assert onp.array_equal((other * 2.0).asarray(), (onp.arange(50) + 1.0) * 2.0)


@pytest.mark.parametrize("nodag", [False, True])
def test_a_forwarded_value_does_not_carry_its_store_back_in_time(oracle_engine, nodag, monkeypatch):
    """Lowering: instructions run in node order and a store runs where its node sits.  `t = a*2; b -= a; b[:] = t` with t
    never stored used to attach the last store to the multiplication - in FRONT of the in-place update, which then read the
    new b (found by the DAG fuzzer, seeds 592 / 1660; the statement order alone triggers it, with or without the DAG)."""
    import ramba_b200 as rb
    from ramba_b200 import ramba

    monkeypatch.setattr(ramba, "NO_DAG", nodag)
    xa, xb = onp.arange(204, dtype=onp.float64).reshape(12, 17), onp.ones((12, 17))
    a, b = rb.fromarray(xa), rb.fromarray(xb)
    rb.sync()
    t = a * 2.0
    b -= a
    b[0:12, 0:17] = t
    del t
    assert onp.array_equal(b.asarray(), xa * 2.0)
    # the same with a reader of the old value in between, and with the sin / cos pairing moving a store up
    a, b = rb.fromarray(xa), rb.fromarray(xb)
    c = rb.fromarray(xb * 3.0)
    rb.sync()
    t = a * 2.0
    u = b + 1.0          # reads the old b
    b[:, :] = t
    del t
    assert onp.array_equal(u.asarray(), xb + 1.0) and onp.array_equal(b.asarray(), xa * 2.0)
    s = rb.sin(a)
    y = c * 2.0          # reads the old c ...
    c[:, :] = rb.cos(a)  # ... before its overwrite by the half SINCOS would like to store early
    rb.sync()
    assert onp.array_equal(y.asarray(), xb * 6.0)
    assert onp.allclose(c.asarray(), onp.cos(xa), rtol=1e-13, atol=1e-15) and onp.allclose(s.asarray(), onp.sin(xa), rtol=1e-13, atol=1e-15)
