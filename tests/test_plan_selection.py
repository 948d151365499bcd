"""Which kernel the CUDA library picks for an op list, checked WITHOUT a GPU through rb200_describe_plan (the planner
runs on the host): the BASELINE programs must land on the specialised kernels - the stencil on the TMA-staged term
kernel, affine maps + sums and column sums on the streaming kernel - and everything outside the lean vocabulary on
the general interpreter, in the form the launch would take."""
import numpy as onp
import pytest


@pytest.fixture
def plans(oracle_engine):
    import _oracle_backend

    del _oracle_backend.PLANS[:]
    return _oracle_backend.PLANS


def _last(plans, prefix):
    hits = [p for p in plans if p.startswith(prefix)]
    assert hits, plans
    return dict(kv.split("=", 1) for kv in hits[-1].split() if "=" in kv)


def test_laplacian_runs_on_the_term_kernel_with_tma(plans):
    import ramba_b200 as rb

    n = 132  # rows of 132 floats: 16-byte multiples, like 1024
    U = rb.fromarray(onp.random.RandomState(0).rand(40, 70, n).astype(onp.float32))
    V = rb.zeros((40, 70, n), dtype=onp.float32)
    rb.sync()
    del plans[:]
    V[1:-1, 1:-1, 1:-1] = (U[:-2, 1:-1, 1:-1] + U[2:, 1:-1, 1:-1] + U[1:-1, :-2, 1:-1] + U[1:-1, 2:, 1:-1]
                           + U[1:-1, 1:-1, :-2] + U[1:-1, 1:-1, 2:] - 6.0 * U[1:-1, 1:-1, 1:-1])
    rb.sync()
    d = _last(plans, "kernel=stencil_terms")
    # (halos are counted from the first staged view, U[:-2, 1:-1, 1:-1]: two planes ahead, one row / column either side)
    assert d["staged_views"] == "7" and d["halo"] == "z0+2,y1+1,x1+1" and d["loader"] == "tma" and d["ring"] == "5"
    assert d["terms"] == "7(f32:6)" and d["direct_views"] == "1"


def test_odd_rows_use_the_cooperative_loader(plans):
    import ramba_b200 as rb

    U = rb.fromarray(onp.random.RandomState(0).rand(9, 35, 131).astype(onp.float32))
    V = rb.zeros((9, 35, 131), dtype=onp.float32)
    rb.sync()
    V[1:-1, 1:-1, 1:-1] = U[:-2, 1:-1, 1:-1] + U[2:, 1:-1, 1:-1] - 2.0 * U[1:-1, 1:-1, 1:-1]
    rb.sync()
    assert _last(plans, "kernel=stencil_terms")["loader"] == "cp.async"


def test_map_reduce_and_streaming_forms(plans):
    import ramba_b200 as rb

    X = rb.fromarray(onp.ones((64, 4096), dtype=onp.float32))
    Y = rb.fromarray(onp.ones((64, 4096), dtype=onp.float32) * 2)
    v = rb.fromarray(onp.ones(4096, dtype=onp.float32))
    rb.sync()
    del plans[:]
    s = (X * 2.0 + 1.0).sum()  # one source, scalar map, global sum: the map + reduce kernel
    d = _last(plans, "kernel=mapred mode=global")
    assert d["source"] == "f32" and d["ops"] == "3(f32:0)" and d["loads"] == "128bit"
    assert float(s) == 3.0 * 64 * 4096
    del plans[:]
    r = (X + v).sum(axis=0)  # row-split matrix + row-broadcast vector, column sums
    rb.sync()
    d = _last(plans, "kernel=mapred mode=columns")
    assert d["broadcast_operand"] == "1" and d["ops"] == "1(f32:1)"
    assert onp.array_equal(r.asarray(), onp.full(4096, 128.0, dtype=onp.float32))
    del plans[:]
    t = (X * Y - 0.5).sum()  # two sources: the streaming term kernel (staged ring)
    d = _last(plans, "kernel=stream_terms mode=elementwise")
    assert d["staged_views"] == "2" and d["reds"] == "1" and int(d["ring_depth"]) >= 3
    assert float(t) == 1.5 * 64 * 4096
    del plans[:]
    Z = X * 3.0 - Y  # elementwise with a store
    rb.sync()
    d = _last(plans, "kernel=stream_terms mode=elementwise")
    assert d["staged_views"] == "2" and d["reds"] == "0"
    assert Z is not None


def test_everything_else_stays_on_the_general_interpreter(plans):
    import ramba_b200 as rb

    a = rb.arange(5000)
    b = (a * 3 + 1) % 7
    rb.sync()
    assert any(p.startswith("kernel=general_interpreter") for p in plans)
    del plans[:]
    c = rb.sin(a * 0.001)
    rb.sync()
    assert all(p.startswith("kernel=general_interpreter") for p in plans), plans
    assert b is not None and c is not None


def test_general_interpreter_forms(plans):
    import ramba_b200 as rb

    x = onp.arange(64 * 4096, dtype=onp.int64).reshape(64, 4096)
    X = rb.fromarray(x)
    Y = rb.fromarray(onp.arange(4 * 16 * 2048, dtype=onp.int64).reshape(4, 16, 2048))
    rb.sync()
    del plans[:]
    r = X.sum(axis=0)  # integer column sums over [rows][2 * 2048 columns]: the 1-D kernel with column accumulators
    rb.sync()
    d = _last(plans, "kernel=general_interpreter form=axis_as_1d")
    assert d["ndim"] == "2" and int(d["ctas"]) > 0 and int(d["smem"]) > 0
    assert onp.array_equal(r.asarray(), x.sum(axis=0))
    del plans[:]
    s = Y.sum(axis=1)  # the reduced dim is not the outermost one: 3-D after the permutation, the general axis kernel
    rb.sync()
    assert _last(plans, "kernel=general_interpreter form=axis_reduce")["ndim"] == "3"
    assert s is not None
    del plans[:]
    Z = X[:, 1:] * 3 + 1  # N-d integer map whose rows fill their tiles: tiles cut along the rows
    rb.sync()
    d = _last(plans, "kernel=general_interpreter form=elementwise")
    assert d["ndim"] == "2" and d["tiling"] == "row"
    assert Z is not None


def test_describe_plan_is_thread_safe(oracle_engine, monkeypatch):
    """rb200_describe_plan keeps its plan per call: threads describing different op lists at the same time (ctypes
    releases the GIL) each get what that op list gets when described alone."""
    import threading

    import ramba_b200 as rb
    from ramba_b200 import _cabi
    from ramba_b200.runtime import RT

    fops = []
    be = RT.backend
    run = be.run

    def record(fop, stream=None):
        fops.append(_cabi.FusedOp.from_buffer_copy(fop))
        return run(fop, stream)

    monkeypatch.setattr(be, "run", record)
    X = rb.fromarray(onp.ones((64, 4096), dtype=onp.float32))
    Y = rb.fromarray(onp.ones((64, 4096), dtype=onp.float32) * 2)
    v = rb.fromarray(onp.ones(4096, dtype=onp.float32))
    rb.sync()
    del fops[:]
    float((X * Y - 0.5).sum())
    float((X * 2.0 + 1.0).sum())
    Z = X * 3.0 - Y
    W = (X + v).sum(axis=0)
    rb.sync()
    assert Z is not None and W is not None
    want = [_cabi.describe_plan(f) for f in fops]
    kernels = {w.split()[0] for w in want}
    assert {"kernel=stream_terms", "kernel=mapred"} <= kernels, want
    bad = []

    def worker(k):
        for i in range(2000):
            j = (k + i) % len(fops)
            got = _cabi.describe_plan(fops[j])
            if got != want[j]:
                bad.append((want[j], got))

    threads = [threading.Thread(target=worker, args=(k,)) for k in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not bad, bad[:3]
