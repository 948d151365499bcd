"""The pending fused op keeps one record per array it touches, and nothing keys arrays by gid outside it.

Structure (read from the package's source): deferred_op keeps no per-gid containers beside its records, bdarray has no
gid registry, and no condition tests `flex_dist` and `remote_constructed` together (flex_dist implies not
remote_constructed, so each such test equals one flag).  Behaviour, on the NumPy oracle (whose values come out right
either way, so the tests look at the flushes): the elided temporary of a map + reduce never reaches memory, and a
statement that reads its own destination through another view is split by a temporary."""
import ast
import os

import numpy as onp
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(HERE, "..", "ramba_b200")


def _modules():
    for name in sorted(os.listdir(PKG)):
        if name.endswith(".py"):
            with open(os.path.join(PKG, name)) as f:
                yield name, ast.parse(f.read(), name)


def _ramba():
    return dict(_modules())["ramba.py"]


def _class(tree, name):
    return [n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == name][0]


_OLD_CONTAINERS = {"use_gids", "read_arrs", "write_arrs", "read_gids", "write_gids", "preconstructed_gids", "keepalives",
                   "elide_gids", "delete_gids"}
_REGISTRY = {"gid_map", "get_by_gid", "valid_gid"}


def test_the_fused_op_keeps_no_per_gid_containers():
    fuser = _class(_ramba(), "deferred_op")
    stored = {n.attr for n in ast.walk(fuser) if isinstance(n, ast.Attribute) and isinstance(n.ctx, ast.Store)}
    assert not stored & _OLD_CONTAINERS, stored & _OLD_CONTAINERS
    assert "add_gid" not in {f.name for f in fuser.body if isinstance(f, ast.FunctionDef)}


def test_no_gid_registry():
    bd = _class(_ramba(), "bdarray")
    names = {t.id for n in bd.body if isinstance(n, ast.Assign) for t in n.targets if isinstance(t, ast.Name)}
    names |= {f.name for f in bd.body if isinstance(f, ast.FunctionDef)}
    assert not names & _REGISTRY, names & _REGISTRY
    for name, tree in _modules():
        used = {n.attr for n in ast.walk(tree) if isinstance(n, ast.Attribute)}
        assert not used & (_REGISTRY | _OLD_CONTAINERS), (name, used & (_REGISTRY | _OLD_CONTAINERS))


def test_no_condition_tests_both_partition_flags():
    for name, tree in _modules():
        for node in ast.walk(tree):
            if isinstance(node, ast.BoolOp):
                attrs = {n.attr for n in ast.walk(node) if isinstance(n, ast.Attribute)}
                assert not {"flex_dist", "remote_constructed"} <= attrs, (name, node.lineno, ast.unparse(node))


def _flushes(monkeypatch):
    """Record the view gids and the op list of every flush."""
    from ramba_b200 import ramba

    flushes = []
    orig = ramba.run_deferred_ops

    def spy(views, prog, *args, **kwargs):
        flushes.append(([g for (g, _) in views], prog))
        return orig(views, prog, *args, **kwargs)

    monkeypatch.setattr(ramba, "run_deferred_ops", spy)
    return flushes


@pytest.mark.parametrize("no_dag", [True, False], ids=["no_dag", "dag"])
def test_the_temporary_of_a_map_reduce_is_never_stored(oracle_engine, monkeypatch, no_dag):
    """`(X*2.0 + 1.0).sum()`: the sum's operand is elided, so the one flush reads X, accumulates into the partial array
    through a reduction slot and stores nothing; the temporary has no view."""
    import ramba_b200 as rb
    from ramba_b200 import _cabi, ramba

    monkeypatch.setattr(ramba, "NO_DAG", no_dag)
    x = rb.fromarray(onp.arange(1000, dtype=onp.float32))
    rb.sync()
    flushes = _flushes(monkeypatch)
    s = float((x * 2.0 + 1.0).sum())  # (not inside the assert: its rewriting would keep the temporaries alive)
    assert s == float((onp.arange(1000, dtype=onp.float32) * 2.0 + 1.0).sum(dtype=onp.float64))
    assert len(flushes) == 1
    gids, prog = flushes[0]
    assert len(gids) == 2 and gids[0] == x.gid, gids
    assert [i for i in prog.insns if i["st_view"] != _cabi.NOSTORE] == []


@pytest.mark.parametrize("no_dag", [True, False], ids=["no_dag", "dag"])
def test_a_statement_reading_its_destination_through_another_view_goes_through_a_temporary(oracle_engine, monkeypatch,
                                                                                           no_dag):
    """`a[1:] = a[:-1]` (alias check 2 on the statement's own operands): the value is stored to a temporary in a flush of
    its own, so no flush reads and writes one array through two different views."""
    import ramba_b200 as rb
    from ramba_b200 import ramba

    monkeypatch.setattr(ramba, "NO_DAG", no_dag)
    a = rb.fromarray(onp.arange(100, dtype=onp.float64))
    rb.sync()
    flushes = _flushes(monkeypatch)
    a[1:] = a[:-1]
    rb.sync()
    exp = onp.arange(100, dtype=onp.float64)
    exp[1:] = exp[:-1].copy()
    assert onp.array_equal(a.asarray(), exp)
    assert len(flushes) == 2 and all(gids.count(a.gid) == 1 for (gids, _) in flushes), flushes
