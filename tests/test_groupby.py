"""groupby: grouped sum, prod, min, max, count, mean, nanmean, var and std along one axis, and `gb OP rhs`.

CPU: the engine through the NumPy restatement of the kernel (_group_vm) against NumPy for every aggregate, source dtype,
axis position and view kind; label forms and errors; gloo worlds 2, 3, 4 and 8 against world 1 in both layouts, with the
transfer counters; the restatement against a per-element brute force; the plan and argument checks of the C-ABI.
GPU: rb200_group_reduce against the restatement bit for bit in every form, and the NumPy cases through the CUDA library."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as onp
import pytest

import _group_vm as GV
import _group_worker as GW

HERE = os.path.dirname(os.path.abspath(__file__))
AGGS = GW.AGGS


@pytest.fixture
def group_engine():
    import _oracle_backend
    from ramba_b200 import ramba
    from ramba_b200.runtime import RT

    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()
    _oracle_backend.install()
    yield
    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()


def expected(x, dim, labels, G, agg):
    """NumPy per group, with the documented values for an empty group."""
    xs = onp.moveaxis(onp.asarray(x), dim, -1)
    out = []
    for g in range(G):
        m = labels == g
        v = xs[..., m]
        with onp.errstate(all="ignore"):
            if agg == "count":
                r = onp.full(v.shape[:-1], m.sum(), dtype=onp.int64)
            elif agg in ("sum", "prod"):
                r = (v.sum(-1) if agg == "sum" else v.prod(-1)).astype(x.dtype)
            elif agg in ("min", "max"):
                if m.any():
                    r = v.min(-1) if agg == "min" else v.max(-1)
                elif x.dtype.kind == "f":
                    r = onp.full(v.shape[:-1], onp.inf if agg == "min" else -onp.inf, dtype=x.dtype)
                else:
                    info = onp.iinfo(x.dtype)
                    r = onp.full(v.shape[:-1], info.max if agg == "min" else info.min, dtype=x.dtype)
            elif agg == "nanmean":
                v64 = v.astype(onp.float64)
                r = onp.nansum(v64, -1) / (~onp.isnan(v64)).sum(-1)
            else:
                v64 = v.astype(onp.float64)
                n = m.sum()
                mean = v64.sum(-1) / n
                var = ((v64 - mean[..., None]) ** 2).sum(-1) / n
                r = {"mean": mean, "var": var, "std": onp.sqrt(var)}[agg]
        out.append(onp.asarray(r))
    return onp.moveaxis(onp.stack(out, -1), -1, dim)


def _close(got, exp, exact):
    if got.shape != exp.shape or got.dtype != exp.dtype:
        return False
    if exact or got.dtype.kind != "f":
        return onp.array_equal(got, exp, equal_nan=True)
    tol = 1e-12 if got.dtype == onp.float64 else 1e-6
    return onp.allclose(got, exp, rtol=tol, atol=0, equal_nan=True)


def _data(shape, dtype, seed):
    x = onp.random.default_rng(seed).integers(-9, 10, size=shape)
    return x.astype(dtype) * (onp.array(0.5, dtype) if onp.dtype(dtype).kind == "f" else 1)


VIEWS = [
    ("plain", (6, 40), lambda x: x, 1),
    ("first_axis", (40, 6), lambda x: x, 0),
    ("middle", (3, 40, 5), lambda x: x, 1),
    ("columns", (30, 70), lambda x: x, 0),
    ("sliced", (9, 50), lambda x: x[1:8, 3:43], 1),
    ("stepped", (9, 90), lambda x: x[::2, ::2], 1),
    ("reversed", (5, 40), lambda x: x[:, ::-1], 1),
    ("transposed", (40, 7), lambda x: x.T, 1),
    ("broadcast", (1, 40), lambda x: onp.broadcast_to(x, (4, 40)) if isinstance(x, onp.ndarray) else x.broadcast_to((4, 40)), 1),
    ("lazy", (6, 40), lambda x: x * 2 + 1, 1),
]


def _case(rb, shape, view, dim, dtype, G=7, seed=0, form="numpy", local_border=0):
    x = _data(shape, dtype, seed)
    hv = view(x)
    labels = onp.random.default_rng(seed + 1).integers(0, G - 1, size=hv.shape[dim])  # group G-1 stays empty
    A = view(rb.fromarray(x, local_border=local_border))
    lab = {"numpy": labels, "list": labels.tolist(), "ramba": rb.fromarray(labels)}[form]
    return A, hv, A.groupby(dim, lab, G), labels


def _check_views(rb, dtypes):
    for name, shape, view, dim in VIEWS:
        for dt in dtypes:
            A, hv, gb, labels = _case(rb, shape, view, dim, dt)
            for agg in AGGS:
                got = getattr(gb, agg)().asarray()
                exp = expected(hv, dim, labels, 7, agg)
                exact = agg in ("sum", "prod", "min", "max", "count") or onp.dtype(dt).kind != "f"
                assert _close(got, exp, exact and agg not in ("mean", "var", "std", "nanmean")), (name, dt, agg, got, exp)


def test_aggregates_match_numpy_every_dtype_and_view(group_engine):
    import ramba_b200 as rb

    _check_views(rb, (onp.float64, onp.float32, onp.int64, onp.int32))


def test_label_forms_num_groups_and_padding(group_engine):
    import ramba_b200 as rb

    for form in ("numpy", "list", "ramba"):
        A, hv, gb, labels = _case(rb, (5, 33), lambda x: x, 1, onp.float64, G=9, form=form)
        assert onp.array_equal(gb.group_array, labels) and gb.num_groups == 9 and gb.dim == 1 and gb.array_to_group is A
        assert _close(gb.sum().asarray(), expected(hv, 1, labels, 9, "sum"), True)
    x = _data((4, 12), onp.float64, 3)
    gb = rb.fromarray(x).groupby(1, onp.arange(12) % 5)
    assert gb.num_groups == 5 and _close(gb.max().asarray(), expected(x, 1, onp.arange(12) % 5, 5, "max"), True)
    A, hv, gb, labels = _case(rb, (8, 21), lambda x: x, 1, onp.float64, local_border=1)
    assert _close(gb.min().asarray(), expected(hv, 1, labels, 7, "min"), True)
    assert _close(gb.var().asarray(), expected(hv, 1, labels, 7, "var"), False)


def test_nanmean_skips_nan(group_engine):
    import ramba_b200 as rb

    x = _data((4, 30), onp.float64, 4)
    x[1, ::3] = onp.nan
    x[2, :] = onp.nan
    labels = onp.arange(30) % 4
    got = rb.fromarray(x).groupby(1, labels, 5).nanmean().asarray()
    assert _close(got, expected(x, 1, labels, 5, "nanmean"), False)
    assert onp.isnan(got[2]).all() and onp.isnan(got[:, 4]).all()


def test_binops(group_engine):
    import ramba_b200 as rb

    x = _data((5, 40), onp.float64, 6)
    labels = onp.random.default_rng(2).integers(0, 6, size=40)
    A = rb.fromarray(x)
    gb = A.groupby(1, labels, 6)
    m = expected(x, 1, labels, 6, "mean")
    assert onp.allclose((gb - gb.mean()).asarray(), x - m[:, labels], rtol=1e-12)
    r = _data((5, 6), onp.float64, 7)
    for name, f in (("__add__", onp.add), ("__mul__", onp.multiply), ("__truediv__", onp.true_divide), ("__gt__", onp.greater)):
        got = getattr(gb, name)(r).asarray()
        exp = f(x, r[:, labels])
        # (true division: the engine's division, as for any two arrays, may differ from NumPy's in the last bit)
        same = onp.allclose(got, exp, rtol=1e-15, atol=0, equal_nan=True) if name == "__truediv__" else onp.array_equal(got, exp)
        assert got.dtype == exp.dtype and same, name
    ri = rb.fromarray(onp.arange(30, dtype=onp.int64).reshape(5, 6))
    got = (gb + ri).asarray()
    assert got.dtype == onp.float64 and onp.array_equal(got, x + onp.arange(30).reshape(5, 6)[:, labels])
    assert onp.array_equal(gb.__rsub__(r).asarray(), r[:, labels] - x)
    with pytest.raises(ValueError):
        gb + onp.zeros((5, 7))


def test_errors(group_engine):
    import ramba_b200 as rb

    A = rb.fromarray(onp.arange(24.0).reshape(4, 6))
    with pytest.raises(IndexError):
        A.groupby(1, [0, 1, 2, 3, 4, 5], 5)
    with pytest.raises(IndexError):
        A.groupby(1, [0, -1, 0, 0, 0, 0], 3)
    with pytest.raises(ValueError):
        A.groupby(1, [0, 1, 0], 3)
    with pytest.raises(ValueError):
        A.groupby(1, onp.zeros(6), 3)
    with pytest.raises(ValueError):
        A.groupby(2, [0] * 6, 3)
    with pytest.raises(ValueError):
        A.groupby(1, [0] * 6, 0)
    with pytest.raises(NotImplementedError):
        A[A > 3.0].groupby(0, [0] * 8, 2)


def test_narrow_integer_and_bool_sources(group_engine):
    """Sources the kernel does not read directly are widened; an empty group's min / max is the dtype's bound."""
    import ramba_b200 as rb

    labels = onp.array([0, 1, 0, 1])
    for dt in (onp.int8, onp.int16, onp.uint8, onp.uint16, onp.uint32, onp.bool_):
        x = (onp.array([[3, 1, 2, 0], [5, 7, 1, 1]]) % (2 if dt == onp.bool_ else 100)).astype(dt)
        gb = rb.fromarray(x).groupby(1, labels, 3)
        for agg in ("min", "max", "sum", "count"):
            got = getattr(gb, agg)().asarray()
            exp = expected(x, 1, labels, 3, agg) if dt != onp.bool_ else None
            if agg in ("min", "max"):
                lo, hi = (False, True) if dt == onp.bool_ else (onp.iinfo(dt).min, onp.iinfo(dt).max)
                assert got.dtype == onp.dtype(dt) and got[:, 2].tolist() == [hi if agg == "min" else lo] * 2, (dt, agg, got)
            if exp is not None:
                assert _close(got, exp, True), (dt, agg, got, exp)
        assert _close(gb.mean().asarray(), expected(x.astype(onp.int64), 1, labels, 3, "mean"), False), dt


def test_empty_grouped_axis_at_one_rank(group_engine):
    import ramba_b200 as rb

    x = onp.zeros((3, 0))
    gb = rb.fromarray(x).groupby(1, onp.zeros(0, dtype=onp.int64), 2)
    assert gb.sum().asarray().tolist() == [[0.0, 0.0]] * 3
    assert gb.prod().asarray().tolist() == [[1.0, 1.0]] * 3
    assert gb.min().asarray().tolist() == [[onp.inf, onp.inf]] * 3
    assert gb.count().asarray().tolist() == [[0, 0]] * 3
    assert onp.isnan(gb.mean().asarray()).all() and onp.isnan(gb.var().asarray()).all() and gb.mean().shape == (3, 2)
    xi = rb.fromarray(onp.zeros((0, 2), dtype=onp.int32)).groupby(0, [], 3)
    assert xi.max().asarray().tolist() == [[onp.iinfo(onp.int32).min] * 2] * 3


# ---- the reference's programs (tests/golden/groupby_golden.npz, made by make_groupby_golden.py) ------------------------
def _golden_tolerance(name, key, ref):
    """Exact: integer results, min / max / count, and sums and means of exactly representable data (every source here
    but the random ones is integers or small multiples of 1/4).  Otherwise rtol 1e-12 in float64; sums of a float32
    source rtol 1e-6 (the reference accumulates float32 in float32, this engine in float64)."""
    agg = key
    if ref.dtype.kind != "f" or agg in ("min", "max", "count"):
        return None
    if name in ("mean_groupby3", "first_axis_season"):
        return 1e-12
    if name == "every_aggregate_float32" and agg in ("sum", "prod", "mean", "var", "std", "final"):
        return 1e-6
    if agg in ("var", "std"):
        return 1e-12
    return None


def _check_groupby_golden():
    import json

    import _groupby_programs

    import ramba_b200 as rb

    z = onp.load(os.path.join(HERE, "golden", "groupby_golden.npz"))
    status = json.loads(str(z["__status__"]))
    assert sorted(status) == sorted(p.__name__ for p in _groupby_programs.PROGRAMS), "regenerate groupby_golden.npz"
    for prog in _groupby_programs.PROGRAMS:
        name = prog.__name__
        assert status[name] == "ok", (name, status[name])
        with onp.errstate(all="ignore"):
            got = prog(rb)
        for k, v in got.items():
            ref = z["%s__%s" % (name, k)]
            tol = _golden_tolerance(name, k, ref)
            assert v.shape == ref.shape and v.dtype == ref.dtype, (name, k, v.dtype, ref.dtype, v.shape, ref.shape)
            if tol is None:
                assert onp.array_equal(v, ref, equal_nan=True), (name, k, v, ref)
            else:
                assert onp.allclose(v, ref, rtol=tol, atol=tol, equal_nan=True), (name, k, v, ref)


def test_reference_groupby_programs(group_engine):
    _check_groupby_golden()


# ---- multi-rank over gloo ---------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run_world(world, out, mode="oracle"):
    port = _free_port()
    procs = []
    for r in range(world):
        env = dict(os.environ)
        env.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r), "MASTER_ADDR": "127.0.0.1",
                    "MASTER_PORT": str(port), "OMP_NUM_THREADS": "1"})
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_group_worker.py"), out, mode], env=env,
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


def _check_worlds(worlds):
    base = worlds[1]
    cuts = set()
    for w, res in worlds.items():
        for k, v in res.items():
            if k.endswith(".counters"):
                continue
            name, agg = k.split(".")[:2]
            cut = bool(res.get("%s.sum.0.counters" % name, [0, 0, 0])[2])
            cuts.add((w > 1, cut))
            # var / std of a cut axis: the squared deviations from an inexact mean are summed in another order
            exact = not (cut and agg in ("var", "std"))
            assert _close(v, base[k], exact) if exact else onp.allclose(v, base[k], rtol=1e-12, equal_nan=True), (w, k)
        for k, c in res.items():
            if not k.endswith(".counters"):
                continue
            agg = k.split(".")[1]
            n_coll, n_bytes, cut, size, is_float = (int(x) for x in c)
            passes = 0 if agg == "count" else (2 if agg in ("var", "std") or (agg == "nanmean" and is_float) else 1)
            if cut:
                assert n_coll == passes and n_bytes == passes * size * 8, (w, k, c)
            else:
                assert n_coll == 0 and n_bytes == 0, (w, k, c)
    assert (True, True) in cuts and (True, False) in cuts, cuts  # both layouts ran at several ranks


@pytest.fixture(scope="module")
def group_worlds(tmp_path_factory):
    d = tmp_path_factory.mktemp("group_worlds")
    return {w: _run_world(w, str(d / ("w%d.npz" % w))) for w in (1, 2, 3, 4, 8)}


@pytest.mark.timeout(1800)
def test_multirank_matches_one_rank(group_worlds):
    _check_worlds(group_worlds)


# ---- the restatement against a per-element brute force ----------------------------------------------------------------
def _brute(x, axis, labels, G, op, C_, center=None):
    src_float = x.dtype.kind == "f"
    acc_t = float if (src_float or op == GV.SQDEV) else int
    L = x.shape[axis]
    O, I = int(onp.prod(x.shape[:axis])), int(onp.prod(x.shape[axis + 1:]))
    x3 = x.reshape(O, L, I)
    out = onp.zeros((O, G, I), dtype=onp.float64 if acc_t is float else onp.int64)
    ident = GV.identity(op, acc_t is float)

    def comb(a, b):
        if op == GV.PROD:
            return a * b
        if op == GV.MIN:
            return b if b < a else a
        if op == GV.MAX:
            return b if b > a else a
        return a + b

    for o in range(O):
        for i in range(I):
            for g in range(G):
                r = onp.float64(ident) if acc_t is float else onp.int64(ident)
                for s0 in range(0, max(L, 1), C_):
                    p = onp.float64(ident) if acc_t is float else onp.int64(ident)
                    for t in range(s0, min(L, s0 + C_)):
                        if labels[t] != g:
                            continue
                        v = x3[o, t, i]
                        if op == GV.SQDEV:
                            d = onp.float64(v) - center[o, g, i]
                            p = p + d * d
                        elif op in (GV.NANSUM, GV.NANCOUNT):
                            if src_float and onp.isnan(v):
                                continue
                            p = p + (1 if op == GV.NANCOUNT else (onp.float64(v) if acc_t is float else onp.int64(v)))
                        else:
                            p = comb(p, onp.float64(v) if acc_t is float else onp.int64(v))
                    r = comb(r, p)
                out[o, g, i] = r
    return out


def test_restatement_against_brute_force():
    rng = onp.random.default_rng(0)
    with onp.errstate(all="ignore"):
        for trial in range(12):
            shape = [int(rng.integers(1, 5)) for _ in range(int(rng.integers(1, 4)))]
            axis = int(rng.integers(0, len(shape)))
            shape[axis] = int(rng.integers(0, 23))
            dt = [onp.float64, onp.float32, onp.int64, onp.int32][trial % 4]
            x = rng.integers(-5, 6, size=shape).astype(dt)
            if x.dtype.kind == "f" and x.size:
                x.reshape(-1)[::5] = onp.nan
            G = int(rng.integers(1, 6))
            labels = rng.integers(0, G, size=shape[axis])
            C_ = int(rng.integers(1, 8))
            for op in range(7):
                O = int(onp.prod(shape[:axis]))
                I = int(onp.prod(shape[axis + 1:]))
                cen = rng.standard_normal(O * G * I).reshape(O, G, I) if op == GV.SQDEV else None
                got = GV.reduce(x, axis, labels, G, op, C_, cen)
                exp = _brute(x, axis, labels, G, op, C_, cen)
                assert onp.array_equal(got, exp, equal_nan=True), (trial, op, shape, axis)


# ---- the C-ABI ---------------------------------------------------------------------------------------------------------
def _view(shape, strides, eb=8, base=0x1000):
    from ramba_b200 import _cabi

    return _cabi.index_view(base, shape, strides, eb)


PLAN_CASES = [  # (shape, strides, axis, G, form)
    ([65536, 3653], [3653, 1], 1, 366, "row"),
    ([65536, 3653], [3653, 1], 1, 4, "row"),
    ([3653, 65536], [65536, 1], 0, 366, "column"),
    ([1 << 28], [1], 0, 16, "row"),
    ([3653, 4096], [1, 3653], 1, 366, "general"),   # transposed
    ([100, 60], [120, 2], 1, 5, "general"),          # stepped
    ([40, 50], [0, 1], 1, 3, "row"),                 # broadcast rows
    ([70, 30, 9], [270, 9, 1], 1, 4, "general"),     # middle axis, short inner run
    ([5, 20000], [20000, 1], 1, 3, "row"),           # too few rows: the axis is split
    ([20000, 3], [3, 1], 0, 2, "general"),
    ([3000, 64], [64, 1], 0, 2, "column"),           # split column form
    ([10, 3000], [3000, 1], 1, 2000, "general"),     # too many groups for the row form
]


def test_describe_group_plan_matches_the_restatement():
    from ramba_b200 import _cabi

    for shape, strides, axis, G, form in PLAN_CASES:
        f = _cabi.group_plan_fields(_cabi.describe_group_plan(_view(shape, strides), axis, G))
        assert f["form"] == form, (shape, strides, axis, G, f)
        assert GV.plan(shape, strides, axis, G) == (form, f["chunk"]), (shape, f)
        L = shape[axis]
        assert f["chunks"] == max(-(-L // f["chunk"]), 1)
    f = _cabi.group_plan_fields(_cabi.describe_group_plan(_view([1 << 28], [1]), 0, 16))
    assert f["chunks"] > 1 and f["scratch"] > 0   # axis split: a fold of the partials in chunk order
    f = _cabi.group_plan_fields(_cabi.describe_group_plan(_view([65536, 3653], [3653, 1]), 1, 4))
    assert f["ctas_per_row"] == 1 and f["cta_chunks"] > 1 and f["scratch"] == 0
    f = _cabi.group_plan_fields(_cabi.describe_group_plan(_view([65536, 3653], [3653, 1]), 1, 366))
    assert f["chunks"] == 1 and f["ctas"] == 65536


def test_malformed_group_arguments_are_rejected():
    from ramba_b200 import _cabi

    lib = _cabi.load()
    P = 0x1000

    def call(view=None, dtype=0, axis=1, G=3, length=6, op=0, center=P, out=P, offsets=P, members=P, scratch=P):
        v = view if view is not None else _view([4, 6], [6, 1])
        t = _cabi.group_table(G, length, offsets, members)
        rc = lib.rb200_group_reduce(C.byref(v), dtype, axis, C.byref(t), op, center, out, scratch, None)
        return rc, lib.rb200_last_error().decode()

    assert "bad op" in call(op=7)[1]
    assert "bad op" in call(op=-1)[1]
    assert "source dtype" in call(dtype=4)[1]
    assert "elem_bytes does not match" in call(dtype=1)[1]
    assert "axis out of range" in call(axis=2)[1]
    assert "axis out of range" in call(axis=-1)[1]
    assert "n_groups must be >= 1" in call(G=0)[1]
    assert "len differs" in call(length=5)[1]
    assert "SQDEV needs center" in call(op=6, center=None)[1]
    assert "null out" in call(out=None)[1]
    assert "null table array" in call(offsets=None)[1]
    assert "null view base pointer" in call(view=_view([4, 6], [6, 1], base=0))[1]
    assert "elem_bytes" in call(view=_view([4, 6], [6, 1], eb=3))[1]
    split = _view([1 << 20], [1])
    assert "null scratch" in call(view=split, axis=0, length=1 << 20, scratch=None)[1]
    assert lib.rb200_describe_group_plan(C.byref(_view([4, 6], [6, 1])), 5, 3) is None
    assert lib.rb200_group_reduce_scratch_bytes(C.byref(_view([4, 6], [6, 1])), 1, 0) < 0
    import torch

    if not torch.cuda.is_available():
        assert "no usable CUDA device" in call()[1]


def test_group_structs_match_the_header(tmp_path):
    from ramba_b200 import _cabi

    src = tmp_path / "layout.c"
    src.write_text(r"""
#include <stdio.h>
#include <stddef.h>
#include "ramba_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %d %d\n", sizeof(rb200_group_table), offsetof(rb200_group_table, len), offsetof(rb200_group_table, offsets),
         offsetof(rb200_group_table, members), RB200_GROUP_SQDEV, RB200_ABI_VERSION);
  return 0;
}
""")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(HERE, "..", "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).decode().split()]
    T = _cabi.GroupTable
    assert got == [C.sizeof(T), T.len.offset, T.offsets.offset, T.members.offset, _cabi.GROUP_SQDEV, _cabi.ABI_VERSION]


def test_group_kernels_do_not_spill():
    """ptxas -v of rb200_group.cu (written by the build): no kernel spills to local memory."""
    log = os.path.join(HERE, "..", "ramba_b200", "csrc", "build", "rb200_group.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("library not built here")
    import re

    text = open(log).read()
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert spills and all(a == "0" and b == "0" for a, b in spills), spills
    assert text.count("Compiling entry function") == len(spills)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def _gpu_vs_vm(shape, strides, axis, G, labels, dt, ops=range(7), pad=16, seed=0):
    """One view of device memory through rb200_group_reduce and the restatement: the same bits for every op."""
    import torch

    from ramba_b200 import _cabi

    dev = torch.device("cuda", 0)
    rng = onp.random.default_rng(seed)
    lo = sum(min(0, (s - 1) * st) for s, st in zip(shape, strides))
    hi = sum(max(0, (s - 1) * st) for s, st in zip(shape, strides))
    nmem = hi - lo + 1 + 2 * pad
    host = rng.standard_normal(nmem) * 4 if onp.dtype(dt).kind == "f" else rng.integers(-1 << 20, 1 << 20, size=nmem)
    host = host.astype(dt)
    if onp.dtype(dt).kind == "f":
        host[::17] = onp.nan
    code = {onp.dtype(onp.float64): 0, onp.dtype(onp.float32): 1, onp.dtype(onp.int64): 2, onp.dtype(onp.int32): 3}[onp.dtype(dt)]
    eb = onp.dtype(dt).itemsize
    d_mem = torch.from_numpy(host.copy()).to(dev)
    base_off = (pad - lo) * eb
    view = _cabi.index_view(d_mem.data_ptr() + base_off, shape, strides, eb, (d_mem.data_ptr(), d_mem.data_ptr() + nmem * eb))
    h_view = _cabi.index_view(host.ctypes.data + base_off, shape, strides, eb)
    L = shape[axis]
    cnt = onp.bincount(labels, minlength=G)
    offs = onp.concatenate([[0], onp.cumsum(cnt)]).astype(onp.int64)
    mem = onp.argsort(labels, kind="stable").astype(onp.int64)
    mem1 = mem if len(mem) else onp.zeros(1, onp.int64)
    d_offs, d_members = torch.from_numpy(offs).to(dev), torch.from_numpy(mem1).to(dev)
    table = _cabi.group_table(G, L, d_offs.data_ptr(), d_members.data_ptr())
    h_table = _cabi.group_table(G, L, offs.ctypes.data, mem1.ctypes.data)
    n_out = int(onp.prod(shape[:axis] + shape[axis + 1:])) * G
    nbytes = _cabi.group_reduce_scratch_bytes(view, axis, G)
    scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    center = rng.standard_normal(max(n_out, 1))
    d_center = torch.from_numpy(center).to(dev)
    form = _cabi.group_plan_fields(_cabi.describe_group_plan(view, axis, G))["form"]
    for op in ops:
        acc_dt = onp.float64 if (onp.dtype(dt).kind == "f" or op == GV.SQDEV) else onp.int64
        d_out = torch.full((max(n_out, 1),), 7, dtype=torch.float64 if acc_dt == onp.float64 else torch.int64, device=dev)
        _cabi.group_reduce(view, code, axis, table, op, d_center.data_ptr(), d_out.data_ptr(), scratch.data_ptr())
        h_out = onp.zeros(max(n_out, 1), dtype=acc_dt)
        GV.group_reduce(h_view, code, axis, h_table, op, center.ctypes.data, h_out.ctypes.data)
        torch.cuda.synchronize()
        got = d_out.cpu().numpy()[:n_out]
        assert got.view(onp.uint64 if acc_dt == onp.float64 else onp.int64).tolist() == \
            h_out[:n_out].view(onp.uint64 if acc_dt == onp.float64 else onp.int64).tolist(), (shape, strides, axis, G, dt, op, form)
    return form


@pytest.mark.gpu
def test_cuda_kernel_matches_the_restatement_every_form():
    rng = onp.random.default_rng(9)
    forms = set()
    layouts = [  # (shape, strides, axis, G)
        ([37, 301], [301, 1], 1, 366),      # row, G > len: empty groups
        ([200, 517], [517, 1], 1, 4),       # row, several chunks per CTA
        ([3, 5000], [5000, 1], 1, 3),       # row, axis split over CTAs (ragged)
        ([1], [1], 0, 1),                   # G = 1, one element
        ([9000], [1], 0, 5),                # 1-D, axis split
        ([301, 70], [70, 1], 0, 9),         # column
        ([2100, 33], [33, 1], 0, 2),        # column, split
        ([60, 41], [1, 60], 1, 6),          # transposed: general
        ([30, 90], [-90, 2], 1, 4),         # reversed rows, stepped axis: general
        ([20, 31, 7], [217, 7, 1], 1, 5),   # middle axis, short inner run: general
        ([12, 40], [0, 1], 1, 3),           # broadcast rows
        ([5, 40, 3, 4], [480, 12, 4, 1], 1, 1),
    ]
    for shape, strides, axis, G in layouts:
        labels = rng.integers(0, G, size=shape[axis])
        if G > 2:
            labels[labels == G - 1] = 0  # the last group stays empty
        for dt in (onp.float64, onp.float32, onp.int64, onp.int32):
            forms.add(_gpu_vs_vm(shape, strides, axis, G, labels, dt))
    assert forms == {"row", "column", "general"}


@pytest.mark.gpu
def test_cuda_kernel_past_2_to_the_31():
    """One f32 source of more than 2^31 elements (64-bit offsets), rows grouped on the last axis, SUM and MAX."""
    import torch

    from ramba_b200 import _cabi

    if torch.cuda.get_device_properties(0).total_memory < (16 << 30):
        pytest.skip("needs 16 GB")
    rows, L = 65540, 32768  # 2^31 + 131072 elements
    dev = torch.device("cuda", 0)
    src = torch.ones(rows * L, dtype=torch.float32, device=dev)
    src[-L:] = torch.arange(L, dtype=torch.float32, device=dev)
    labels = onp.arange(L) % 3
    offs = onp.concatenate([[0], onp.cumsum(onp.bincount(labels))]).astype(onp.int64)
    mem = onp.argsort(labels, kind="stable").astype(onp.int64)
    d_offs, d_mem = torch.from_numpy(offs).to(dev), torch.from_numpy(mem).to(dev)
    view = _cabi.index_view(src.data_ptr(), [rows, L], [L, 1], 4, (src.data_ptr(), src.data_ptr() + src.numel() * 4))
    table = _cabi.group_table(3, L, d_offs.data_ptr(), d_mem.data_ptr())
    out = torch.zeros(rows * 3, dtype=torch.float64, device=dev)
    scratch = torch.empty(max(_cabi.group_reduce_scratch_bytes(view, 1, 3), 1), dtype=torch.uint8, device=dev)
    _cabi.group_reduce(view, 1, 1, table, GV.SUM, None, out.data_ptr(), scratch.data_ptr())
    got = out.view(rows, 3).cpu().numpy()
    last = onp.arange(L, dtype=onp.float64)
    assert onp.array_equal(got[-1], [last[labels == g].sum() for g in range(3)])
    assert onp.array_equal(got[0], onp.bincount(labels).astype(onp.float64))
    _cabi.group_reduce(view, 1, 1, table, GV.MAX, None, out.data_ptr(), scratch.data_ptr())
    assert onp.array_equal(out.view(rows, 3).cpu().numpy()[-1], [last[labels == g].max() for g in range(3)])
    del src
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_cuda_aggregates_match_numpy(gpu_engine):
    import ramba_b200 as rb

    _check_views(rb, (onp.float64, onp.float32, onp.int64, onp.int32))
    test_nanmean_skips_nan(None)
    test_binops(None)
    test_label_forms_num_groups_and_padding(None)


@pytest.mark.gpu
def test_cuda_reference_programs_and_edges(gpu_engine):
    _check_groupby_golden()
    test_narrow_integer_and_bool_sources(None)
    test_empty_grouped_axis_at_one_rank(None)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_cuda_world2_over_nccl(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    one = _run_world(1, str(tmp_path / "w1.npz"), "cuda")
    two = _run_world(2, str(tmp_path / "w2.npz"), "cuda")
    _check_worlds({1: one, 2: two})
