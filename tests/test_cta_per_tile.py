"""The lean 1-D interpreter kernel's grid: one CTA per tile (`grid=cta_per_tile` in rb200_describe_plan) instead of a
persistent grid walking tiles b, b+grid, ...  Which launches get it, checked without a GPU; that RB200_NO_CTA_PER_TILE=1
(read once per process: a subprocess) restores the walk; and, on the GPU, that both grids give the same bits - every
element is computed by the same thread of its tile either way."""
import os
import re
import subprocess
import sys

import numpy as onp
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
TILE = 256 * 8
N = TILE * 1000 + 5  # more tiles than any persistent grid of 2 CTAs per SM


@pytest.fixture
def plans(oracle_engine):
    import _oracle_backend

    del _oracle_backend.PLANS[:]
    return _oracle_backend.PLANS


def _ctas(p):
    return int(re.search(r" ctas=(\d+)", p).group(1))


def test_the_headline_chain_runs_one_cta_per_tile(plans):
    import ramba_b200 as rb

    A = rb.arange(N) / 1000.0
    rb.sync()
    del plans[:]
    B = rb.sin(A)
    C = rb.cos(A)
    D = B * B + C ** 2
    rb.sync()
    interp = [p for p in plans if p.startswith("kernel=general_interpreter form=elementwise")]
    assert interp and all(" grid=cta_per_tile " in p and p.endswith(" variant=lean") for p in interp), plans
    assert all(_ctas(p) == (N + TILE - 1) // TILE for p in interp), plans
    assert onp.max(onp.abs(D.asarray() - 1.0)) <= 4 * onp.finfo(onp.float64).eps


def test_other_launches_keep_the_walk(plans):
    import ramba_b200 as rb

    A = rb.arange(N) / 1000.0
    rb.sync()
    del plans[:]
    s = rb.sin(A).sum()  # a reduction: not the lean kernel
    rb.sync()
    assert float(s) == pytest.approx(float(onp.sin(onp.arange(N) / 1000.0).sum()))
    assert plans and not any("grid=cta_per_tile" in p for p in plans), plans
    X = rb.fromarray(onp.arange(N, dtype=onp.float64).reshape(5, -1)[:, 1:])
    Y = rb.sin(X) * 2.0  # a 2-D op list
    rb.sync()
    assert Y.shape == X.shape
    assert all(("grid=cta_per_tile" in p) == ("variant=lean" in p) for p in plans), plans


def _plans_with(env):
    code = """import sys; sys.path[:0] = [%r, %r]
import _oracle_backend
from ramba_b200.runtime import RT
RT.reset()
_oracle_backend.install()
import ramba_b200 as rb
A = rb.arange(%d) / 1000.0
rb.sync()
B = rb.sin(A); C = rb.cos(A); D = B * B + C ** 2
rb.sync()
print("\\n".join(_oracle_backend.PLANS))
""" % (ROOT, HERE, N)
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-3000:]
    return [p for p in out.stdout.split("\n") if p.startswith("kernel=general_interpreter form=elementwise")]


def test_the_kill_switch_restores_the_walk():
    lean = [p for p in _plans_with({"RB200_NO_CTA_PER_TILE": "1"}) if p.endswith(" variant=lean")]
    assert lean and not any("grid=" in p for p in lean), lean
    assert all(_ctas(p) < (N + TILE - 1) // TILE for p in lean), lean


def test_the_full_interpreter_keeps_the_walk():
    interp = _plans_with({"RB200_NO_LEAN_INTERP": "1"})
    assert interp and not any("variant=lean" in p or "grid=" in p for p in interp), interp


# ---- GPU: one CTA per tile against the walk, bit for bit --------------------------------------------------------------
SIZES = [TILE * 64, TILE * 37 + 1, TILE * 1000 + 5, 1000]


def _walk_worker(out_dir):
    """Every program of test_lean_interpreter at every size on the walking grid (run under RB200_NO_CTA_PER_TILE=1)."""
    import test_lean_interpreter as t

    for p in t.PROGRAMS:
        for n in SIZES:
            outs, plans = t._run(p, n)
            assert plans and not any("grid=cta_per_tile" in q for q in plans), plans
            for i, o in enumerate(outs):
                onp.save(os.path.join(out_dir, "%s_%d_%d.npy" % (p, n, i)), o)


@pytest.mark.gpu
def test_one_cta_per_tile_and_the_walk_give_the_same_bits(gpu_engine, tmp_path):
    import test_lean_interpreter as t

    code = "import sys; sys.path[:0] = [%r, %r]; import test_cta_per_tile as t; t._walk_worker(%r)" % (ROOT, HERE, str(tmp_path))
    walk = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, RB200_NO_CTA_PER_TILE="1"), capture_output=True, text=True, timeout=1200)
    assert walk.returncode == 0, walk.stdout[-2000:] + walk.stderr[-3000:]
    for p in t.PROGRAMS:
        for n in SIZES:
            outs, plans = t._run(p, n)
            interp = [q for q in plans if q.startswith("kernel=general_interpreter")]
            assert interp and all(" grid=cta_per_tile " in q for q in interp), (p, n, plans)
            for i, o in enumerate(outs):
                ref = onp.load(os.path.join(str(tmp_path), "%s_%d_%d.npy" % (p, n, i)))
                assert o.dtype == ref.dtype and o.shape == ref.shape, (p, n, i)
                assert o.tobytes() == ref.tobytes(), (p, n, i, int(onp.sum(o.view(onp.uint8) != ref.view(onp.uint8))))
