"""The statement seam between the array API, the DAG and the fuser, and the one table of reductions.

Structure (read from the package's source): every statement reaches the DAG and the fuser as one `Statement` record, the
entry points take no reference-era code arguments, and no module but program.py translates between reduction names and
kernel codes.  Values: the reduction table, written out.  Behaviour: a statement inside the fuser's pending op holds no
array handle, only ArrRefs, whether it came straight from the API call (RAMBA_NO_DAG=1) or through the DAG."""
import ast
import gc
import os
import re
import types

import numpy as onp
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(HERE, "..", "ramba_b200")


def _modules():
    for name in sorted(os.listdir(PKG)):
        if name.endswith(".py"):
            with open(os.path.join(PKG, name)) as f:
                src = f.read()
            yield name, src, ast.parse(src, name)


def _methods(tree, cls_name):
    for node in ast.walk(tree):
        if isinstance(node, ast.ClassDef) and node.name == cls_name:
            return {f.name: f for f in node.body if isinstance(f, ast.FunctionDef)}
    raise AssertionError("no class " + cls_name)


def _params(f):
    a = f.args
    return [p.arg for p in a.posonlyargs + a.args + a.kwonlyargs]


def test_statement_entry_points_take_no_code_arguments():
    tree = dict((n, t) for n, _, t in _modules())["ramba.py"]
    dag, fuser = _methods(tree, "DAG"), _methods(tree, "deferred_op")
    assert "add" not in dag
    entry = [dag["assign"], dag["reduce"], dag["_add"], fuser["add_op"]]
    for f in entry:
        assert not {"imports", "precode", "postcode", "oplist", "write_array", "_reads"} & set(_params(f)), f.name
    assert _params(fuser["add_op"]) == ["cls", "stmt"]
    smap = [n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "smap"][0]
    assert "imports" in _params(smap)  # (smap's public argument is the reference's, and stays)


def test_no_scalar_temporary_remains():
    for name, src, _ in _modules():
        assert not re.search(r"\b(TempVar|temp_var|get_temp_var)\b", src), name


def test_only_program_maps_reduction_codes_to_names():
    def is_red(n):
        return isinstance(n, ast.Attribute) and n.attr.startswith("RED_")

    hits = []
    for name, _, tree in _modules():
        if name == "program.py":
            continue
        for node in ast.walk(tree):
            if isinstance(node, ast.Dict) and any(is_red(x) for x in list(node.keys) + list(node.values) if x is not None):
                hits.append((name, node.lineno))
    assert not hits, hits


def test_every_statement_is_a_record():
    """No call hands the DAG or the fuser a `[dst, expr]` list, and the fuser is given exactly one record."""
    seam = {"add", "add_op", "assign", "reduce"}
    for name, _, tree in _modules():
        for node in ast.walk(tree):
            if not (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr in seam):
                continue
            recv = ast.unparse(node.func.value)
            if node.func.attr == "add_op":
                assert len(node.args) == 1 and not node.keywords, (name, node.lineno)
            elif not recv.endswith("DAG"):
                continue
            assert not any(isinstance(a, ast.List) for a in node.args), (name, node.lineno)


# ---- the reduction table ----------------------------------------------------------------------------------------------
_DTYPES = [onp.bool_, onp.int8, onp.int32, onp.int64, onp.uint8, onp.float32, onp.float64]
_INF = float("inf")
# op: (kernel code (include/ramba_b200.h rb200_redop), combine operator, all-reduce op, identity per dtype in _DTYPES order)
_TABLE = {
    "sum": (0, "add", "SUM", [0, 0, 0, 0, 0, 0, 0]),
    "prod": (1, "mul", "PRODUCT", [1, 1, 1, 1, 1, 1, 1]),
    "min": (2, "min", "MIN", [True, 127, 2147483647, 9223372036854775807, 255, _INF, _INF]),
    "max": (3, "max", "MAX", [False, -128, -2147483648, -9223372036854775808, 0, -_INF, -_INF]),
    "all": (1, "mul", "MIN", [1, 1, 1, 1, 1, 1, 1]),
    "any": (0, "add", "MAX", [0, 0, 0, 0, 0, 0, 0]),
}


@pytest.mark.parametrize("op", sorted(_TABLE))
def test_reduction_table(op):
    import torch
    from ramba_b200.program import REDUCTIONS, red_identity

    code, combine, allreduce, idents = _TABLE[op]
    red = REDUCTIONS[op]
    assert (red.code, red.combine, red.allreduce, red.truth) == (code, combine, allreduce, op in ("all", "any"))
    for dt, want in zip(_DTYPES, idents):
        got = red_identity(op, dt)
        assert type(got) is type(want) and got == want, (op, dt, got)
    stack = torch.tensor([[3, 0, 5], [1, 1, 7]], dtype=torch.int64)
    folded = {"sum": [4, 1, 12], "prod": [3, 0, 35], "min": [1, 0, 5], "max": [3, 1, 7], "all": [1, 0, 5], "any": [3, 1, 7]}
    assert red.fold(stack).tolist() == folded[op]


def test_reduction_fill_and_mask_values(oracle_engine, monkeypatch):
    """all / any fill their partial array with a bool; a masked-out element contributes the int identity."""
    import ramba_b200 as rb
    from ramba_b200 import ramba

    fills = []
    orig = ramba._fill_now
    monkeypatch.setattr(ramba, "_fill_now", lambda nd, v: (fills.append(v), orig(nd, v))[1])
    a = rb.fromarray(onp.array([True, False, True]))
    assert not a.all() and a.any() and int(rb.fromarray(onp.arange(4)).min()) == 0
    assert [(type(v), v) for v in fills] == [(bool, True), (bool, False), (int, 9223372036854775807)]


# ---- no handles in the pending op ---------------------------------------------------------------------------------------
def _reachable_handles(roots):
    """ndarray handles reachable from `roots` through object references (classes, modules and functions not followed)."""
    from ramba_b200.ramba import ndarray

    seen, todo, found = set(), list(roots), []
    while todo:
        x = todo.pop()
        if id(x) in seen or isinstance(x, (type, types.ModuleType, types.FunctionType, types.MethodType)):
            continue
        seen.add(id(x))
        if isinstance(x, ndarray):
            found.append(x)
            continue
        todo.extend(gc.get_referents(x))
        if hasattr(type(x), "__slots__"):
            todo.extend(getattr(x, s) for s in type(x).__slots__ if s != "__weakref__" and hasattr(x, s))
    return found


@pytest.mark.parametrize("no_dag", [True, False], ids=["no_dag", "dag"])
def test_pending_statements_hold_no_handles(oracle_engine, monkeypatch, no_dag):
    import ramba_b200 as rb
    from ramba_b200 import ramba

    monkeypatch.setattr(ramba, "NO_DAG", no_dag)
    x = rb.fromarray(onp.arange(64, dtype=onp.float64))
    rb.sync()
    y = x * 2.0
    if not no_dag:
        ramba.DAG.execute_all()  # (hands every pending statement to the fuser without flushing)
    cur = ramba.deferred_op.ramba_deferred_ops
    assert cur is not None and len(cur.statements) == 1
    st = cur.statements[0]
    assert isinstance(st, ramba.Statement) and st.reads is None
    assert isinstance(st.dst, ramba.ArrRef) and st.dst.gid == y.gid
    assert _reachable_handles(cur.statements) == []
    assert onp.array_equal(y.asarray(), onp.arange(64) * 2.0)
