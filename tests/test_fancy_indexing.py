"""Integer-array indexing (`a[idx]`, `a[idx] = v`) and `random.choice`.

CPU: every case of _index_worker against NumPy at one rank (all stored dtypes, host and ramba index arrays) and over gloo
at worlds 2, 3, 4 and 8; errors; ordering with pending statements; launch count; the NumPy restatement of the kernels
(_index_vm) against a per-element brute force; argument checks of the C-ABI.  GPU: rb200_gather / rb200_scatter /
rb200_route against the restatement bit for bit, and the cases through the CUDA library."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as onp
import pytest

import _index_vm as V
import _index_worker as IW

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture
def index_engine():
    import _oracle_backend
    from ramba_b200 import ramba
    from ramba_b200.runtime import RT

    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()
    _oracle_backend.install()
    yield
    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()


def _check_cases(dtypes, forms):
    import ramba_b200 as rb

    for name, shape, view, index in IW.cases():
        for dt in dtypes:
            for form in forms:
                g, e, ga, ea = IW.run_case(rb, name, shape, view, index, dt, form)
                assert g.shape == e.shape and g.dtype == e.dtype and onp.array_equal(g, e), (name, dt, form)
                assert ga.dtype == ea.dtype and onp.array_equal(ga, ea), (name, dt, form, "write")


def test_cases_match_numpy_every_dtype(index_engine):
    _check_cases(IW.DTYPES, ("numpy", "list", "ramba"))


def test_padded_source(index_engine):
    import ramba_b200 as rb

    g, e, ga, ea = IW.run_case(rb, "adjacent", (5, 6, 7), lambda x: x, lambda mk: (slice(None), mk(onp.array([5, 0])), 3),
                               onp.float64, "ramba", local_border=1)
    assert onp.array_equal(g, e) and onp.array_equal(ga, ea)


def _golden():
    import json

    z = onp.load(os.path.join(HERE, "golden", "fancy_golden.npz"))
    return z, json.loads(str(z["__status__"]))


def _check_golden():
    """Every program of _fancy_programs against the outputs of the reference (tests/golden/make_fancy_golden.py)."""
    import _fancy_programs

    import ramba_b200 as rb

    z, status = _golden()
    assert sorted(status) == sorted(p.__name__ for p in _fancy_programs.PROGRAMS), "regenerate fancy_golden.npz"
    for prog in _fancy_programs.PROGRAMS:
        name = prog.__name__
        assert status[name] == "ok", (name, status[name])
        got = prog(rb)
        for k, v in got.items():
            ref = z["%s__%s" % (name, k)]
            assert v.shape == ref.shape and onp.array_equal(v, ref), (name, k)
    sh = z["fancy_indexing1__shapes"]
    assert sh.tolist() == [[3, 3, 0, 0, 0], [1, 4, 3, 41, 0], [2, 3, 1, 1, 5]]


def test_reference_fancy_indexing_programs(index_engine):
    _check_golden()


def test_errors(index_engine):
    import ramba_b200 as rb

    a = onp.arange(24.0).reshape(4, 6)
    A = rb.fromarray(a)
    with pytest.raises(IndexError, match="axis 1 with size 6"):
        A[:, [0, 6]]
    before = A.asarray().tobytes()
    with pytest.raises(IndexError, match="axis 0 with size 4"):
        A[rb.fromarray(onp.array([1, -5])), 2] = 3.0
    with pytest.raises(IndexError, match="axis 0 with size 4"):
        A[rb.fromarray(onp.array([2, 4]))]
    assert A.asarray().tobytes() == before
    with pytest.raises(IndexError):
        A[onp.array([0.0, 1.0])]
    with pytest.raises(IndexError):
        A[rb.fromarray(onp.array([0.0]))]
    with pytest.raises(IndexError):
        A[onp.array([True, False, True, False]), 1]
    with pytest.raises(NotImplementedError):
        A[A > 3.0][[0, 1]]
    with pytest.raises(NotImplementedError):
        A[A > 3.0][[0, 1]] = 1.0
    assert A.asarray().tobytes() == before
    # an empty result still checks ramba index arrays (NumPy: np.zeros((4, 0, 3))[[7]] raises)
    Z = rb.zeros((4, 0, 3))
    with pytest.raises(IndexError, match="axis 0 with size 4"):
        Z[rb.fromarray(onp.array([7]))]
    with pytest.raises(IndexError, match="axis 0 with size 4"):
        Z[rb.fromarray(onp.array([7]))] = 1.0
    # host index arrays of a dtype the engine does not store
    assert A[onp.array([1, 3], dtype=onp.uint64), 0].asarray().tolist() == [6.0, 18.0]
    A[onp.array([2], dtype=onp.uint64), 1] = 5.0
    assert A.asarray()[2, 1] == 5.0


@pytest.mark.parametrize("mode", ["dag", "no_dag", "verify_plan", "verify_lower"])
def test_ordering_with_pending_statements(mode, tmp_path):
    """A pending write to the source is seen by the gather; a pending read of the target sees the old values."""
    env = dict(os.environ)
    env.update({"no_dag": {"RAMBA_NO_DAG": "1"}, "verify_plan": {"RB200_VERIFY_PLAN_CACHE": "1"},
                "verify_lower": {"RB200_VERIFY_LOWER_CACHE": "1"}}.get(mode, {}))
    code = r"""
import sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import numpy as onp
import _oracle_backend
_oracle_backend.install()
import ramba_b200 as rb
for rep in range(2):
    a = rb.fromarray(onp.arange(10.0))
    a[2:5] = -1.0                     # pending write to the source
    g = a[[3, 8, 2]].asarray()
    assert g.tolist() == [-1.0, 8.0, -1.0], g
    t = a * 2                         # pending read of the target, t alive
    a[rb.fromarray(onp.array([0, 9]))] = 100.0
    assert t.asarray().tolist() == [0.0, 2.0, -2.0, -2.0, -2.0, 10.0, 12.0, 14.0, 16.0, 18.0], t.asarray()
    assert a.asarray().tolist() == [100.0, 1.0, -1.0, -1.0, -1.0, 5.0, 6.0, 7.0, 8.0, 100.0]
    a[[1, 2]] += 1
    assert a.asarray()[:3].tolist() == [100.0, 2.0, 0.0]
print("ok")
""" % (os.path.join(HERE, ".."), HERE)
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    assert out.returncode == 0 and "ok" in out.stdout, out.stdout + out.stderr


def test_one_rank_read_launches(index_engine):
    """The address-stream op list (lin and its out-of-range count), the fill of that count's accumulator, the gather."""
    import ramba_b200 as rb
    from ramba_b200.runtime import RT

    A = rb.fromarray(onp.arange(1000.0))
    c = rb.fromarray(onp.arange(999, -1, -3))
    rb.sync()
    n0 = RT.launches
    r = A[c]
    assert RT.launches - n0 == 3
    assert onp.array_equal(r.asarray(), onp.arange(1000.0)[onp.arange(999, -1, -3)])


def test_choice(index_engine):
    import ramba_b200 as rb

    pool = onp.arange(50.0) * 3
    g1, g2 = rb.random.default_rng(4), rb.random.default_rng(4)
    got = g1.choice(pool, size=(7, 9)).asarray()
    idx = g2.integers(0, 50, (7, 9)).asarray()
    assert onp.array_equal(got, pool[idx])
    assert g1._state._draws == g2._state._draws == 1
    assert onp.array_equal(g1.choice(pool, 5).asarray(), g2.choice(rb.fromarray(pool), 5).asarray())
    rs1, rs2 = rb.random.RandomState(8), rb.random.RandomState(8)
    assert onp.array_equal(rs1.choice(30, 11).asarray(), rs2.randint(0, 30, 11).asarray())
    rb.random.seed(3)
    x = rb.random.choice(pool, 6).asarray()
    rb.random.seed(3)
    assert onp.array_equal(x, pool[rb.random.randint(0, 50, 6).asarray()])
    with pytest.raises(NotImplementedError):
        g1.choice(pool, 3, replace=False)
    with pytest.raises(NotImplementedError):
        g1.choice(pool, 3, p=onp.full(50, 0.02))


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
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_index_worker.py"), out, mode], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=400)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, o))
    for rc, o in outs:
        assert rc == 0, o[-3000:]
    return dict(onp.load(out))


@pytest.fixture(scope="module")
def index_worlds(tmp_path_factory):
    d = tmp_path_factory.mktemp("index_worlds")
    return {w: _run_world(w, str(d / ("w%d.npz" % w))) for w in (1, 2, 3, 4, 8)}


def _check_world_results(worlds):
    base = worlds[1]
    for w, res in worlds.items():
        for k in res:
            if k.endswith((".read", ".write", "view_write")):
                assert res[k].dtype == res[k + "_exp"].dtype and onp.array_equal(res[k], res[k + "_exp"]), (w, k)
        assert onp.array_equal(res["choice"], base["choice"]) and onp.array_equal(res["choice_int"], base["choice_int"]), w
        if w > 1:
            assert res["stats"][0] > 0 and res["stats"][1] > 0, w


@pytest.mark.timeout(1200)
def test_multirank_matches_numpy(index_worlds):
    _check_world_results(index_worlds)


# ---- the restatement against a per-element brute force ----------------------------------------------------------------
def _buf(a):
    return a.ctypes.data


def test_restatement_against_brute_force():
    from ramba_b200 import _cabi

    rng = onp.random.default_rng(0)
    for trial in range(30):
        k = int(rng.integers(1, 4))
        shape = [int(rng.integers(1, 6)) for _ in range(k)]
        strides = [int(rng.integers(-7, 8)) for _ in range(k)]
        mem = rng.integers(0, 1 << 62, size=400).astype(onp.uint64)
        base_idx = 200
        view = _cabi.index_view(_buf(mem) + base_idx * 8, shape, strides, 8)
        size = int(onp.prod(shape))
        lin = rng.integers(-2, size + 2, size=37).astype(onp.int64)
        out = onp.zeros(37, dtype=onp.uint64)
        bad = onp.zeros(1, dtype=onp.uint64)
        V.gather(view, _buf(lin), 37, _buf(out), _buf(bad))
        nbad = 0
        for i, l in enumerate(lin):
            if not 0 <= l < size:
                nbad += 1
                assert out[i] == 0
                continue
            c = onp.unravel_index(int(l), shape)
            assert out[i] == mem[base_idx + sum(int(c[d]) * strides[d] for d in range(k))]
        assert int(bad[0]) == nbad
    # route: a random grid of 2-D cells with random owners and offsets
    for trial in range(20):
        shape = [int(rng.integers(2, 9)), int(rng.integers(2, 9))]
        cuts = [sorted({0, shape[d]} | set(int(x) for x in rng.integers(1, shape[d], size=2))) for d in range(2)]
        ncell = (len(cuts[0]) - 1) * (len(cuts[1]) - 1)
        owners = rng.integers(0, 3, size=ncell)
        offs = rng.integers(0, 1000, size=ncell)
        st = rng.integers(-5, 6, size=(ncell, 2))
        table, keep = _cabi.route_table(shape, cuts, owners, offs, st, 3)
        n = 50
        lin = rng.integers(-1, shape[0] * shape[1] + 1, size=n).astype(onp.int64)
        o_off, o_slot, o_cnt, bad = onp.zeros(n, onp.int64), onp.zeros(n, onp.int64), onp.zeros(3, onp.int64), onp.zeros(1, onp.uint64)
        V.route(table, _buf(lin), n, _buf(o_off), _buf(o_slot), _buf(o_cnt), _buf(bad))
        groups = {r: [] for r in range(3)}
        for i, l in enumerate(lin):
            if not 0 <= l < shape[0] * shape[1]:
                assert o_slot[i] == -1
                continue
            y, x = divmod(int(l), shape[1])
            j0 = max(j for j in range(len(cuts[0]) - 1) if cuts[0][j] <= y)
            j1 = max(j for j in range(len(cuts[1]) - 1) if cuts[1][j] <= x)
            cell = j0 * (len(cuts[1]) - 1) + j1
            groups[int(owners[cell])].append((i, int(offs[cell]) + (y - cuts[0][j0]) * int(st[cell, 0]) + (x - cuts[1][j1]) * int(st[cell, 1])))
        order = [e for r in range(3) for e in groups[r]]
        assert o_cnt.tolist() == [len(groups[r]) for r in range(3)]
        for s, (i, off) in enumerate(order):
            assert o_slot[i] == s and o_off[s] == off
        assert int(bad[0]) == sum(1 for l in lin if not 0 <= l < shape[0] * shape[1])


def test_index_kernels_do_not_spill():
    """ptxas -v of rb200_index.cu (written by the build): no kernel spills to local memory."""
    log = os.path.join(HERE, "..", "ramba_b200", "csrc", "build", "rb200_index.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("library not built here")
    import re

    text = open(log).read()
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert spills and all(a == "0" and b == "0" for a, b in spills), spills
    assert text.count("Compiling entry function") == len(spills)


# ---- the C-ABI ---------------------------------------------------------------------------------------------------------
def test_index_structs_match_the_header(tmp_path):
    from ramba_b200 import _cabi

    src = tmp_path / "layout.c"
    src.write_text(r"""
#include <stdio.h>
#include <stddef.h>
#include "ramba_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu\n", sizeof(rb200_index_view), offsetof(rb200_index_view, shape), offsetof(rb200_index_view, stride),
         offsetof(rb200_index_view, alloc_lo), offsetof(rb200_index_view, elem_bytes));
  printf("%zu %zu %zu %zu %zu\n", sizeof(rb200_route_table), offsetof(rb200_route_table, n_cells), offsetof(rb200_route_table, cut_start),
         offsetof(rb200_route_table, cuts), offsetof(rb200_route_table, cell_stride));
  return 0;
}
""")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(HERE, "..", "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).decode().split()]
    IV, RTb = _cabi.IndexView, _cabi.RouteTable
    assert got == [C.sizeof(IV), IV.shape.offset, IV.stride.offset, IV.alloc_lo.offset, IV.elem_bytes.offset,
                   C.sizeof(RTb), RTb.n_cells.offset, RTb.cut_start.offset, RTb.cuts.offset, RTb.cell_stride.offset]


def test_malformed_index_arguments_are_rejected():
    """Rejected with a reason before any device query (so this holds on a machine without a GPU)."""
    from ramba_b200 import _cabi

    lib = _cabi.load()
    P = 0x1000

    def gat(v, n=4, lin=P, out=P, bad=P):
        return lib.rb200_gather(C.byref(v), lin, n, out, bad, None), lib.rb200_last_error().decode()

    def sca(v, n=4, lin=P, vals=P, bad=P):
        return lib.rb200_scatter(C.byref(v), lin, n, vals, bad, None), lib.rb200_last_error().decode()

    ok = dict(base=P, shape=[4, 4], strides=[4, 1], elem_bytes=8)

    def view(**kw):
        d = dict(ok)
        d.update(kw)
        return _cabi.index_view(d["base"], d["shape"], d["strides"], d["elem_bytes"], d.get("bounds"))

    for call in (gat, sca):
        assert "elem_bytes must be 1, 2, 4 or 8" in call(view(elem_bytes=3))[1]
        v6 = view()
        v6.ndim = 6
        assert "ndim out of range" in call(v6)[1]
        assert "null view base pointer" in call(view(base=0))[1]
        assert "view outside its allocation" in call(view(bounds=(P, P + 8 * 15)))[1]
        assert "null pointer" in call(view(), lin=0)[1]
        assert "negative n" in call(view(), n=-1)[1]
        assert call(view(), n=0)[0] == 0  # nothing to do
    t, keep = _cabi.route_table([8], [[0, 4, 8]], [0, 1], [0, 0], [[1], [1]], 2)

    def rou(t):
        return lib.rb200_route(C.byref(t), P, 4, P, P, P, P, P, None), lib.rb200_last_error().decode()

    t2, keep2 = _cabi.route_table([8], [[0, 4, 7]], [0, 1], [0, 0], [[1], [1]], 2)
    assert "not a grid" in rou(t2)[1]
    t3, keep3 = _cabi.route_table([8], [[0, 5, 4, 8]], [0, 1, 0], [0, 0, 0], [[1], [1], [1]], 2)
    assert "not a grid" in rou(t3)[1]
    t4, keep4 = _cabi.route_table([8], [[0, 4, 8]], [0, 1], [0, 0], [[1], [1]], 65)
    assert "too many ranks" in rou(t4)[1]
    t5, keep5 = _cabi.route_table([8], [[0, 4, 8]], [0, 2], [0, 0], [[1], [1]], 2)
    assert "cell owner out of range" in rou(t5)[1]
    import torch

    if not torch.cuda.is_available():
        assert "no usable CUDA device" in rou(t)[1]


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_cuda_kernels_match_the_restatement():
    import torch

    from ramba_b200 import _cabi

    dev = torch.device("cuda", 0)
    rng = onp.random.default_rng(1)
    layouts = [([1000], [1]), ([37, 41], [41, 1]), ([6, 7, 9], [63, 9, 1]), ([41, 37], [1, 41]), ([50], [-3]),
               ([9, 11], [15, 1])]  # flat, 2-D, 3-D, transposed, negative stride, padded rows
    for eb, np_dt in ((1, onp.uint8), (2, onp.uint16), (4, onp.uint32), (8, onp.uint64)):
        for shape, strides in layouts:
            size = int(onp.prod(shape))
            lo = sum(min(0, (s - 1) * st) for s, st in zip(shape, strides))
            hi = sum(max(0, (s - 1) * st) for s, st in zip(shape, strides))
            pad = 64
            nmem = hi - lo + 1 + 2 * pad
            host = rng.integers(0, 1 << min(8 * eb, 62), size=nmem, dtype=onp.uint64).astype(np_dt)
            for n in (0, 1, 7, 1001):
                lin = rng.integers(0, size, size=n).astype(onp.int64)
                if n >= 7:
                    lin[1], lin[5] = -1, size  # counted and skipped
                d_mem = torch.from_numpy(host.copy().view(onp.uint8)).to(dev)
                base_off = (pad - lo) * eb
                bounds = (d_mem.data_ptr(), d_mem.data_ptr() + d_mem.numel())
                view = _cabi.index_view(d_mem.data_ptr() + base_off, shape, strides, eb, bounds)
                d_lin = torch.from_numpy(lin).to(dev)
                d_out = torch.zeros(max(n, 1) * eb, dtype=torch.uint8, device=dev)
                d_bad = torch.zeros(1, dtype=torch.int64, device=dev)
                _cabi.gather(view, d_lin.data_ptr(), n, d_out.data_ptr(), d_bad.data_ptr())
                h_mem = host.copy()
                h_view = _cabi.index_view(h_mem.ctypes.data + base_off, shape, strides, eb)
                h_out = onp.zeros(max(n, 1), dtype=np_dt)
                h_bad = onp.zeros(1, dtype=onp.uint64)
                V.gather(h_view, lin.ctypes.data, n, h_out.ctypes.data, h_bad.ctypes.data)
                torch.cuda.synchronize()
                assert onp.array_equal(d_out.cpu().numpy().view(np_dt)[:n], h_out[:n]), (eb, shape, n)
                assert int(d_bad.cpu()[0]) == int(h_bad[0])
                # scatter with distinct targets; the bytes around the view stay as they were
                lin_u = rng.permutation(size)[:min(n, size)].astype(onp.int64)
                m = len(lin_u)
                if m >= 7:
                    lin_u[2] = -1
                vals = rng.integers(0, 1 << min(8 * eb, 62), size=max(m, 1), dtype=onp.uint64).astype(np_dt)
                d_bad.zero_()
                d_lin_u, d_vals = torch.from_numpy(lin_u).to(dev), torch.from_numpy(vals).to(dev)
                _cabi.scatter(view, d_lin_u.data_ptr(), m, d_vals.data_ptr(), d_bad.data_ptr())
                h_bad[:] = 0
                V.scatter(h_view, lin_u.ctypes.data, m, vals.ctypes.data, h_bad.ctypes.data)
                torch.cuda.synchronize()
                assert onp.array_equal(d_mem.cpu().numpy().view(np_dt), h_mem), (eb, shape, n, "scatter")
                assert int(d_bad.cpu()[0]) == int(h_bad[0])


@pytest.mark.gpu
def test_cuda_route_matches_the_restatement():
    import torch

    from ramba_b200 import _cabi

    dev = torch.device("cuda", 0)
    rng = onp.random.default_rng(2)
    for n in (0, 1, 33, 5000, 200001):
        shape = [300, 70]
        cuts = [[0, 100, 250, 300], [0, 35, 70]]
        owners = rng.integers(0, 5, size=6)
        offs = rng.integers(0, 10 ** 6, size=6)
        st = rng.integers(-100, 100, size=(6, 2))
        table, keep = _cabi.route_table(shape, cuts, owners, offs, st, 5)
        lin = rng.integers(-3, 21003, size=n).astype(onp.int64)
        h = [onp.zeros(max(n, 1), onp.int64), onp.zeros(max(n, 1), onp.int64), onp.zeros(5, onp.int64), onp.zeros(1, onp.uint64)]
        V.route(table, lin.ctypes.data, n, h[0].ctypes.data, h[1].ctypes.data, h[2].ctypes.data, h[3].ctypes.data)
        d = [torch.zeros(max(n, 1), dtype=torch.int64, device=dev) for _ in range(2)] + [torch.zeros(5, dtype=torch.int64, device=dev),
                                                                                        torch.zeros(1, dtype=torch.int64, device=dev)]
        scratch = torch.empty(_cabi.route_scratch_bytes(n, 5), dtype=torch.uint8, device=dev)
        d_lin = torch.from_numpy(lin).to(dev)
        _cabi.route(table, d_lin.data_ptr(), n, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(), scratch.data_ptr())
        torch.cuda.synchronize()
        nv = int(h[2].sum())
        assert onp.array_equal(d[2].cpu().numpy(), h[2]), n
        assert onp.array_equal(d[1].cpu().numpy()[:n], h[1][:n]), n
        assert onp.array_equal(d[0].cpu().numpy()[:nv], h[0][:nv]), n
        assert int(d[3].cpu()[0]) == int(h[3][0])


@pytest.mark.gpu
def test_cuda_gather_past_2_to_the_31(gpu_engine):
    """One int8 source of more than 2^31 elements, indexed near its end (64-bit addressing)."""
    import torch

    from ramba_b200 import _cabi

    if torch.cuda.get_device_properties(0).total_memory < (8 << 30):
        pytest.skip("needs 8 GB")
    n_src = (1 << 31) + 4099
    src = torch.empty(n_src, dtype=torch.int8, device="cuda")
    src[-4096:] = torch.arange(4096, device="cuda").to(torch.int8)
    lin = torch.tensor([n_src - 1, n_src - 4096, n_src - 2, (1 << 31) + 5, n_src], dtype=torch.int64, device="cuda")
    out = torch.zeros(5, dtype=torch.int8, device="cuda")
    bad = torch.zeros(1, dtype=torch.int64, device="cuda")
    view = _cabi.index_view(src.data_ptr(), [n_src], [1], 1, (src.data_ptr(), src.data_ptr() + n_src))
    _cabi.gather(view, lin.data_ptr(), 5, out.data_ptr(), bad.data_ptr())
    exp = onp.arange(4096).astype(onp.int8)
    assert out.cpu().numpy().tolist() == [exp[-1], exp[0], exp[-2], exp[(1 << 31) + 5 - (n_src - 4096)], 0]
    assert int(bad.cpu()[0]) == 1
    del src
    torch.cuda.empty_cache()
    # N-d decode with 64-bit division: rows of 65536 int8 padded to 65537, more than 2^32 elements, dims not mergeable
    rows, cols, pitch = 65537, 65536, 65537
    mem = torch.zeros(rows * pitch, dtype=torch.int8, device="cuda")
    picks = [(rows - 1, cols - 1), (rows - 1, 0), (40000, 12345), (0, 7), (65535, 65535)]
    for k, (r, c) in enumerate(picks):
        mem[r * pitch + c] = k + 1
    mem[(rows - 1) * pitch + cols] = 99  # a pad byte, never addressed
    view2 = _cabi.index_view(mem.data_ptr(), [rows, cols], [pitch, 1], 1, (mem.data_ptr(), mem.data_ptr() + mem.numel()))
    lin2 = torch.tensor([r * cols + c for r, c in picks] + [rows * cols], dtype=torch.int64, device="cuda")
    out2 = torch.zeros(len(picks) + 1, dtype=torch.int8, device="cuda")
    bad.zero_()
    _cabi.gather(view2, lin2.data_ptr(), lin2.numel(), out2.data_ptr(), bad.data_ptr())
    assert out2.cpu().numpy().tolist() == [1, 2, 3, 4, 5, 0] and int(bad.cpu()[0]) == 1
    # scatter through the same view, then the bytes written are exactly the addressed ones
    vals = torch.tensor([11, 12], dtype=torch.int8, device="cuda")
    lin3 = torch.tensor([(rows - 1) * cols + cols - 2, 3 * cols + 1], dtype=torch.int64, device="cuda")
    _cabi.scatter(view2, lin3.data_ptr(), 2, vals.data_ptr(), bad.data_ptr())
    assert int(mem[(rows - 1) * pitch + cols - 2]) == 11 and int(mem[3 * pitch + 1]) == 12
    assert int(mem[(rows - 1) * pitch + cols]) == 99 and int((mem != 0).sum()) == len(picks) + 3
    del mem


@pytest.mark.gpu
def test_cuda_unaligned_streams():
    """lin, out and values at odd element offsets take the scalar (non-vector) kernels; same bits as the restatement."""
    import torch

    from ramba_b200 import _cabi

    dev = torch.device("cuda", 0)
    rng = onp.random.default_rng(4)
    for eb, np_dt in ((1, onp.uint8), (2, onp.uint16), (4, onp.uint32), (8, onp.uint64)):
        for shape, strides in (([3001], [1]), ([61, 53], [1, 61])):
            size = int(onp.prod(shape))
            host = rng.integers(0, 1 << min(8 * eb, 62), size=size, dtype=onp.uint64).astype(np_dt)
            n = 2001
            lin = onp.concatenate([[0], rng.integers(0, size, size=n)]).astype(onp.int64)
            lin[7] = -1
            d_mem = torch.from_numpy(host.copy()).to(dev)
            view = _cabi.index_view(d_mem.data_ptr(), shape, strides, eb)
            d_lin = torch.from_numpy(lin).to(dev)
            d_out = torch.zeros(n + 1, dtype=d_mem.dtype, device=dev)
            d_bad = torch.zeros(1, dtype=torch.int64, device=dev)
            _cabi.gather(view, d_lin[1:].data_ptr(), n, d_out[1:].data_ptr(), d_bad.data_ptr())
            h_out = onp.zeros(n, dtype=np_dt)
            h_bad = onp.zeros(1, dtype=onp.uint64)
            hv = host.copy()
            V.gather(_cabi.index_view(hv.ctypes.data, shape, strides, eb), lin[1:].ctypes.data, n, h_out.ctypes.data, h_bad.ctypes.data)
            torch.cuda.synchronize()
            assert onp.array_equal(d_out[1:].cpu().numpy().view(np_dt), h_out), (eb, shape)
            assert int(d_bad.cpu()[0]) == int(h_bad[0])
            tgt = onp.concatenate([[0], rng.permutation(size)[:n]]).astype(onp.int64)
            vals = onp.concatenate([[0], rng.integers(0, 1 << min(8 * eb, 62), size=n, dtype=onp.uint64)]).astype(np_dt)
            d_tgt, d_vals = torch.from_numpy(tgt).to(dev), torch.from_numpy(vals).to(dev)
            _cabi.scatter(view, d_tgt[1:].data_ptr(), n, d_vals[1:].data_ptr(), d_bad.data_ptr())
            V.scatter(_cabi.index_view(hv.ctypes.data, shape, strides, eb), tgt[1:].ctypes.data, n, vals[1:].ctypes.data, h_bad.ctypes.data)
            torch.cuda.synchronize()
            assert onp.array_equal(d_mem.cpu().numpy().view(np_dt), hv), (eb, shape, "scatter")


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_cuda_world2_over_nccl(tmp_path):
    """The multi-rank exchange through the CUDA library: route, counts all-gather and grouped P2P over NCCL."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    one = _run_world(1, str(tmp_path / "w1.npz"), "cuda")
    two = _run_world(2, str(tmp_path / "w2.npz"), "cuda")
    _check_world_results({1: one, 2: two})


@pytest.mark.gpu
def test_cuda_cases_match_numpy(gpu_engine):
    _check_cases(IW.DTYPES, ("numpy", "ramba"))


@pytest.mark.gpu
def test_cuda_reference_programs_and_choice(gpu_engine):
    _check_golden()
    test_choice(None)
    test_one_rank_read_launches(None)
