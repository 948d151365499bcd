"""The lean instantiation of the 1-D general interpreter (rb200_elementwise_lean.cu): which op lists it takes, checked
without a GPU through rb200_describe_plan; that ptxas keeps it out of local memory; and, on the GPU, that it computes
the same bits as the full interpreter kernel (RB200_NO_LEAN_INTERP=1, read once per process: a subprocess)."""
import os
import re
import subprocess
import sys

import numpy as onp
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
TILE = 256 * 8  # elements per tile of the 1-D kernels


@pytest.fixture
def plans(oracle_engine):
    import _oracle_backend

    del _oracle_backend.PLANS[:]
    return _oracle_backend.PLANS


def _interp(plans):
    hits = [p for p in plans if p.startswith("kernel=general_interpreter form=elementwise")]
    assert hits, plans
    return hits


def test_the_headline_chain_plans_lean(plans):
    import ramba_b200 as rb

    A = rb.arange(5000) / 1000.0
    rb.sync()
    del plans[:]
    B = rb.sin(A)
    C = rb.cos(A)
    D = B * B + C ** 2
    rb.sync()
    assert all(p.endswith(" variant=lean") for p in _interp(plans)), plans
    assert onp.max(onp.abs(D.asarray() - 1.0)) <= 4 * onp.finfo(onp.float64).eps


def test_float32_sin_and_a_scalar_operand_plan_lean(plans):
    import ramba_b200 as rb

    X = rb.fromarray(onp.linspace(-3, 3, 5000).astype(onp.float32))
    Y = rb.fromarray(onp.linspace(-3, 3, 5000))
    rb.sync()
    del plans[:]
    S = rb.sin(X)
    T = rb.sin(Y) ** 2 * 2.5 - Y
    rb.sync()
    assert len(_interp(plans)) == 1 and all(p.endswith(" variant=lean") for p in _interp(plans)), plans
    assert S.dtype == onp.float32 and T is not None


def _not_lean(plans, what):
    hits = [p for p in plans if p.startswith("kernel=general_interpreter")]
    assert hits, (what, plans)
    assert not any("variant=lean" in p for p in hits), (what, plans)


def test_what_the_lean_kernel_does_not_take(plans):
    import ramba_b200 as rb

    n = 5000
    A = rb.arange(n) / 1000.0
    I = rb.arange(n) * 3
    B = rb.zeros(n)
    rb.sync()
    cases = [
        ("reduction", lambda: float(rb.sin(A).sum())),
        ("masked store", lambda: B.__setitem__(A > 2.0, rb.sin(A))),
        ("CVT", lambda: rb.sin(A) + I),
        ("integer %", lambda: (I % 7) * rb.sin(A)),
        ("unaligned source", lambda: rb.sin(A[1:])),
        ("strided source", lambda: rb.sin(A[::2])),
        ("IOTA", lambda: rb.sin(rb.arange(n) * 0.001)),
        ("PHILOX", lambda: rb.sin(rb.random.random(n))),
    ]
    for what, run in cases:
        del plans[:]
        r = run()
        rb.sync()
        _not_lean(plans, what)
        assert r is not None or what == "masked store"


def test_the_kill_switch_keeps_everything_on_the_full_kernel():
    code = """
import sys
sys.path[:0] = [%r, %r]
import _oracle_backend
from ramba_b200.runtime import RT
RT.reset()
_oracle_backend.install()
import ramba_b200 as rb
A = rb.arange(5000) / 1000.0
rb.sync()
B = rb.sin(A); C = rb.cos(A); D = B * B + C ** 2
rb.sync()
print("\\n".join(_oracle_backend.PLANS))
""" % (ROOT, HERE)
    env = dict(os.environ, RB200_NO_LEAN_INTERP="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-3000:]
    plans = out.stdout.split("\n")
    assert any(p.startswith("kernel=general_interpreter form=elementwise") for p in plans), plans
    assert not any("variant=lean" in p for p in plans), plans


def test_the_lean_kernel_does_not_spill():
    """ptxas -v of rb200_elementwise_lean.cu (written by the build): no spills, and no local memory but the 40-byte
    table of the CUDA library's large-argument sin / cos reduction (|x| >= 1e9, out of line)."""
    log = os.path.join(ROOT, "ramba_b200", "csrc", "build", "rb200_elementwise_lean.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("library not built here")
    text = open(log).read()
    m = re.search(r"Function properties for _ZN5rb20021vm_elementwise_kernel\w*\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", text)
    assert m, text[-2000:]
    frame, st, ld = (int(g) for g in m.groups())
    assert st == 0 and ld == 0, m.group(0)
    assert frame <= 40, m.group(0)
    assert text.count("Compiling entry function") == 1


# ---- GPU: lean against full, bit for bit ------------------------------------------------------------------------------
SIZES = [TILE * 64, TILE * 37 + 1, 1000]
PROGRAMS = ["chain", "sin", "cos", "sin_f32", "powi", "scalar"]


def _inputs(n):
    rng = onp.random.default_rng(n)
    x = rng.uniform(-50.0, 50.0, n)
    x[::97] *= 1e10  # large arguments: the library's reduction path
    return x


def _run(program, n):
    """The program on the GPU; returns its outputs as NumPy arrays and the plans of its op lists."""
    import ramba_b200 as rb
    from ramba_b200 import _cabi
    from ramba_b200.runtime import RT

    x = _inputs(n)
    X = rb.fromarray(x)
    X32 = rb.fromarray((x % 7.0).astype(onp.float32))
    A = rb.arange(n) / 1000.0
    rb.sync()
    be = RT.be()
    run, plans = be.run, []

    def record(fop, stream=None):
        plans.append(_cabi.describe_plan(fop))
        return run(fop, stream)

    be.run = record
    try:
        if program == "chain":
            B = rb.sin(A)
            C = rb.cos(A)
            outs = [B, C, B * B + C ** 2]
        elif program == "sin":
            outs = [rb.sin(X)]
        elif program == "cos":
            outs = [rb.cos(X)]
        elif program == "sin_f32":
            outs = [rb.sin(X32)]
        elif program == "powi":
            outs = [rb.sin(X) ** 2 + X]
        else:
            outs = [(rb.cos(X) - 0.25) * 3.5 + X]
        rb.sync()
    finally:
        be.run = run
    return [o.asarray() for o in outs], plans


def _full_worker(out_dir):
    """Every (program, size) on the full kernel, outputs saved as .npy (run under RB200_NO_LEAN_INTERP=1)."""
    for p in PROGRAMS:
        for n in SIZES:
            outs, plans = _run(p, n)
            assert plans and not any("variant=lean" in q for q in plans), plans
            for i, o in enumerate(outs):
                onp.save(os.path.join(out_dir, "%s_%d_%d.npy" % (p, n, i)), o)


@pytest.mark.gpu
def test_lean_and_full_give_the_same_bits(gpu_engine, tmp_path):
    code = "import sys; sys.path[:0] = [%r, %r]; import test_lean_interpreter as t; t._full_worker(%r)" % (ROOT, HERE, str(tmp_path))
    env = dict(os.environ, RB200_NO_LEAN_INTERP="1")
    full = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert full.returncode == 0, full.stdout[-2000:] + full.stderr[-3000:]
    for p in PROGRAMS:
        for n in SIZES:
            outs, plans = _run(p, n)
            interp = [q for q in plans if q.startswith("kernel=general_interpreter")]
            assert interp and all(q.endswith(" variant=lean") for q in interp), (p, n, plans)
            for i, o in enumerate(outs):
                ref = onp.load(os.path.join(str(tmp_path), "%s_%d_%d.npy" % (p, n, i)))
                assert o.dtype == ref.dtype and o.shape == ref.shape, (p, n, i)
                assert o.tobytes() == ref.tobytes(), (p, n, i, int(onp.sum(o.view(onp.uint8) != ref.view(onp.uint8))))
