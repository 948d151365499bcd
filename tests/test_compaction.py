"""Stream compaction: nonzero, flatnonzero, argwhere, count_nonzero, extract and compress, and one-argument where.

CPU: the engine through the NumPy restatement of the kernels (_compact_vm) against NumPy with == for every stored dtype,
0-d to 4-d, view kinds, densities, empty arrays, lazy conditions, inputs written after the call, both DAG modes, the
errors and the dispatch; float extract compared bit for bit; gloo worlds 2, 3, 4 and 8 against world 1 with the transfer
counters; the restatement against a brute force at run and chunk edges; the plan and the argument checks of the C-ABI;
no spills.
GPU: rb200_compact_count / rb200_compact against the restatement in every form and dtype and at chunk edges, past 2^31
elements; the NumPy cases through the CUDA library; world 2 over NCCL where two GPUs exist."""
import ctypes as C
import os
import re
import socket
import subprocess
import sys
import types

import numpy as onp
import pytest

import _compact_vm as CV
import _compact_worker as CW

HERE = os.path.dirname(os.path.abspath(__file__))
CV.extend_oracle_backend()  # (also for the oracle stand-in of the -m gpu tests under RB200_DRY_GPU_TESTS)
DTYPES = (onp.float64, onp.float32, onp.int64, onp.int32, onp.bool_, onp.uint8, onp.int8, onp.int16, onp.uint16, onp.uint32)
T = CV.CHUNK


@pytest.fixture
def compact_engine():
    import _oracle_backend
    from ramba_b200 import ramba
    from ramba_b200.runtime import RT

    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()
    _oracle_backend.install()
    yield
    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()


def _data(shape, dtype, seed, density=0.5):
    """Nonzero at about `density`; floats also get -0.0 (zero) and NaN (nonzero)."""
    r = onp.random.default_rng(seed)
    keep = r.random(shape) < density
    x = onp.where(keep, r.integers(1, 5, size=shape), 0)
    if onp.dtype(dtype) == onp.bool_:
        return keep
    x = x.astype(dtype)
    if x.dtype.kind == "f" and x.size > 4:
        f = x.reshape(-1)
        f[r.integers(0, f.size, 3)] = -0.0
        f[r.integers(0, f.size, 2)] = onp.nan
        f[r.integers(0, f.size, 2)] = -2.5
    return x


def _bits(x):
    x = onp.asarray(x)
    return x.view("u%d" % x.dtype.itemsize) if x.dtype.kind == "f" else x


def _same(got, exp, what):
    from ramba_b200 import ndarray

    assert isinstance(got, ndarray), what
    g = got.asarray()
    assert g.dtype == exp.dtype and g.shape == exp.shape and onp.array_equal(_bits(g), _bits(exp)), (what, g, exp)


def _check(rb, hv, A, V=None, hvals=None):
    if hv.ndim == 0:
        with pytest.raises(ValueError, match="0d arrays"):
            rb.nonzero(A)
    else:
        got, exp = rb.nonzero(A), onp.nonzero(hv)
        assert isinstance(got, tuple) and len(got) == len(exp)
        for g, e in zip(got, exp):
            _same(g, e.astype(onp.int64), ("nonzero", hv.dtype, hv.shape))
    _same(rb.flatnonzero(A), onp.flatnonzero(hv).astype(onp.int64), ("flatnonzero", hv.dtype, hv.shape))
    _same(rb.argwhere(A), onp.argwhere(hv).astype(onp.int64), ("argwhere", hv.dtype, hv.shape))
    n = rb.count_nonzero(A)
    assert type(n) is type(onp.count_nonzero(hv)) and n == onp.count_nonzero(hv)
    if V is not None:
        _same(rb.extract(A, V), onp.extract(hv, hvals), ("extract", hv.dtype, hv.shape, hvals.dtype))


SHAPES = [(), (7,), (5, 9), (3, 4, 5), (2, 3, 4, 5)]


def _check_dtypes_and_ranks(rb, dtypes=DTYPES):
    for dt in dtypes:
        for i, shape in enumerate(SHAPES):
            x = _data(shape, dt, i)
            v = _data(shape, dt, i + 50, density=0.9)
            if shape:
                _check(rb, x, rb.fromarray(x), rb.fromarray(v), v)
            else:  # (a 0-d array holds its value in the engine's scalar dtype)
                A, V = rb.array(x), rb.array(v)
                _check(rb, A.asarray(), A, V, V.asarray())


def test_every_dtype_and_rank(compact_engine):
    import ramba_b200 as rb

    _check_dtypes_and_ranks(rb)


VIEWS = [
    ("sliced", (9, 50), lambda x: x[1:8, 3:43]),
    ("stepped", (9, 90), lambda x: x[::2, ::3]),
    ("reversed", (5, 40), lambda x: x[::-1, ::-1]),
    ("transposed", (40, 7), lambda x: x.T),
    ("transposed3", (4, 6, 5), lambda x: x.transpose(2, 0, 1)),
    ("broadcast", (1, 40), lambda x: onp.broadcast_to(x, (4, 40)) if isinstance(x, onp.ndarray) else x.broadcast_to((4, 40))),
    ("lazy", (6, 40), lambda x: x * 2 - 1),
]


def _check_views(rb, dtypes=(onp.float64, onp.float32, onp.int64, onp.int16, onp.uint8)):
    for name, shape, view in VIEWS:
        for dt in dtypes:
            x = _data(shape, dt, 3)
            v = _data(shape, onp.float64, 4, density=1.0)
            _check(rb, onp.asarray(view(x)), view(rb.fromarray(x)), view(rb.fromarray(v)), onp.asarray(view(v)))
    x = _data((12, 10), onp.float64, 4)  # a padded shard
    _check(rb, x[2:9, 1:8], rb.fromarray(x, local_border=2)[2:9, 1:8])


def test_views_and_lazy_inputs(compact_engine):
    import ramba_b200 as rb

    _check_views(rb)


def _check_densities_and_edges(rb):
    for density in (0.0, 0.003, 0.5, 1.0):
        for n in (0, 1, T - 1, T, T + 1, 3 * T + 17):
            x = _data((n,), onp.float64, n, density)
            v = _data((n,), onp.float64, n + 1, 1.0)
            _check(rb, x, rb.fromarray(x), rb.fromarray(v), v)
    x = _data((3, T + 5), onp.uint8, 9, 0.5)  # runs longer than a chunk
    _check(rb, x, rb.fromarray(x), rb.fromarray(x.astype(onp.int16)), x.astype(onp.int16))
    e = rb.zeros((4, 0))
    assert [a.shape for a in rb.nonzero(e)] == [(0,), (0,)] and rb.flatnonzero(e).shape == (0,)
    assert rb.argwhere(e).shape == (0, 2) and rb.extract(e, e).shape == (0,)


def test_densities_empty_arrays_and_chunk_edges(compact_engine):
    import ramba_b200 as rb

    _check_densities_and_edges(rb)


def _check_pending_and_writes(rb):
    x = _data((30, 20), onp.float64, 1)
    A = rb.fromarray(x)
    cond = A > 1.5  # lazy
    idx, vals = rb.flatnonzero(cond), rb.extract(cond, A)
    A[:, :] = 0.0  # written after the call: the results are concrete
    _same(idx, onp.flatnonzero(x > 1.5).astype(onp.int64), "lazy condition")
    _same(vals, onp.extract(x > 1.5, x), "lazy extract")
    B = rb.fromarray(x.copy())
    B[3:5] = 7.0  # a pending write to the input runs first
    y = x.copy()
    y[3:5] = 7.0
    _same(rb.nonzero(B)[1], onp.nonzero(y)[1].astype(onp.int64), "pending write")
    _same(rb.extract(onp.asarray(y > 2), B), onp.extract(y > 2, y), "host condition")


def test_pending_inputs_and_later_writes(compact_engine):
    import ramba_b200 as rb

    _check_pending_and_writes(rb)


def test_without_the_dag(compact_engine, monkeypatch):
    import ramba_b200 as rb
    from ramba_b200 import ramba

    monkeypatch.setattr(ramba, "NO_DAG", True)  # RAMBA_NO_DAG=1: statements go straight to the fuser
    _check_pending_and_writes(rb)
    _check_densities_and_edges(rb)


def _check_errors_and_dispatch(rb):
    x = _data((6, 7), onp.float64, 9)
    X = rb.fromarray(x)
    with pytest.raises(NotImplementedError):
        rb.nonzero(X[X > 3.0])
    with pytest.raises(NotImplementedError, match=re.escape("(6, 7)") + ".*" + re.escape("(7,)")):
        rb.extract(X, X[0])
    with pytest.raises(ValueError):
        rb.compress(onp.ones((2, 2)), X)
    with pytest.raises(onp.exceptions.AxisError):
        X.compress([1, 0], axis=2)
    # NumPy's functions and the methods dispatch here
    for f in ("nonzero", "flatnonzero", "argwhere"):
        r = getattr(onp, f)(X)
        e = getattr(onp, f)(x)
        for g, h in zip(r if isinstance(r, tuple) else (r,), e if isinstance(e, tuple) else (e,)):
            _same(g, h.astype(onp.int64), f)
    for g, h in zip(X.nonzero(), x.nonzero()):
        _same(g, h.astype(onp.int64), "ndarray.nonzero")
    for g, h in zip(rb.where(X), onp.where(x)):
        _same(g, h.astype(onp.int64), "one-argument where")
    assert onp.count_nonzero(X) == onp.count_nonzero(x)
    _same(onp.count_nonzero(X, axis=1), onp.count_nonzero(x, axis=1).astype(onp.int64), "count_nonzero axis")
    _same(rb.count_nonzero(X, axis=0, keepdims=True), onp.count_nonzero(x, axis=0, keepdims=True).astype(onp.int64), "keepdims")
    _same(onp.extract(X > 0, X), onp.extract(x > 0, x), "np.extract")
    # compress: short conditions are padded with False, a True past the end raises
    for c, ax in (([1, 0, 1], 0), ([0, 1, 1, 0, 0, 0, 1], 1), ([1, 0], 1), ([1, 0, 0, 0, 0, 0, 0, 0], 1), ([0, 1, 0, 1], None), ([], 0)):
        exp = onp.compress(c, x, axis=ax)
        _same(rb.compress(c, X, axis=ax), exp, ("compress", c, ax))
        _same(rb.compress(rb.fromarray(onp.array(c, dtype=bool)), X, axis=ax), exp, ("compress ramba", c, ax))
        _same(onp.compress(c, X, axis=ax), exp, ("np.compress", c, ax))
    _same(X.compress([True, False, True], axis=0), onp.compress([1, 0, 1], x, axis=0), "ndarray.compress")
    for c in ([0, 0, 0, 0, 0, 0, 0, 1], [1] * 43):
        with pytest.raises(IndexError):
            rb.compress(c, X, axis=0 if len(c) == 8 else None)
        with pytest.raises(IndexError):
            rb.compress(rb.fromarray(onp.array(c, dtype=bool)), X, axis=0 if len(c) == 8 else None)
    # unchanged: a ramba bool index is a masked view, a NumPy bool index raises
    assert X[X > 0].maskarray is not None
    with pytest.raises(IndexError):
        X[x > 0]


def test_errors_and_dispatch(compact_engine):
    import ramba_b200 as rb

    _check_errors_and_dispatch(rb)


# ---- the restatement against a brute force ------------------------------------------------------------------------------
def _brute(pred, run_len, run_base):
    """Per element, walking run by run and chunk by chunk: (counts, output position of every selected element)."""
    n = pred.size
    n_runs = n // run_len
    cpr = -(-run_len // T)
    counts = onp.zeros(n_runs * cpr, dtype=onp.int64)
    for p in range(n):
        if pred[p]:
            r, o = divmod(p, run_len)
            counts[(o // T) * n_runs + r] += 1
    dest = []
    for r in range(n_runs):
        at = run_base[r]
        for o in range(run_len):
            if pred[r * run_len + o]:
                dest.append(at)
                at += 1
    return counts, onp.array(dest, dtype=onp.int64)


def test_restatement_against_brute_force():
    rng = onp.random.default_rng(0)
    for run_len in (1, 31, 32, T - 1, T, T + 1, 2 * T + 3):
        for n_runs in (1, 3):
            for density in (0.0, 0.01, 0.5, 1.0):
                pred = rng.random(run_len * n_runs) < density
                if n_runs == 3:
                    pred[run_len:2 * run_len] = False  # an empty run
                bases = onp.cumsum(rng.integers(0, 3, n_runs)) * 100 + onp.arange(n_runs) * run_len
                counts = CV.counts_of(pred, run_len)
                incl = CV.inclusive(counts, n_runs)
                exp_c, exp_d = _brute(pred, run_len, bases)
                assert onp.array_equal(counts, exp_c), (run_len, n_runs, density)
                sel, dest = CV.destinations(pred, run_len, counts, incl, bases)
                assert onp.array_equal(sel, onp.flatnonzero(pred)) and onp.array_equal(dest, exp_d), (run_len, n_runs, density)


# ---- the C-ABI ----------------------------------------------------------------------------------------------------------
def _view(shape, strides, eb=1, base=0x1000, bounds=None):
    from ramba_b200 import _cabi

    return _cabi.index_view(base, shape, strides, eb, bounds)


PLAN_CASES = [  # (shape, strides, run_len)
    ([1 << 30], [1], 1 << 30),
    ([32768, 32768], [32768, 1], 32768 * 32768),
    ([32768, 16384], [32768, 1], 16384),    # a column half of a (32768, 32768) array: runs of 4 chunks
    ([1000, 3], [3, 1], 3),                 # short runs: many per CTA
    ([4096, 1], [1, 1], 1),
    ([300, 70], [1, 300], 70 * 300),        # transposed: strided loads
]


def test_describe_compact_plan_matches_the_restatement():
    from ramba_b200 import _cabi

    for shape, strides, run_len in PLAN_CASES:
        f = _cabi.group_plan_fields(_cabi.describe_compact_plan(_view(shape, strides), run_len))
        n = int(onp.prod(shape))
        assert (f["runs"], f["chunks_per_run"], f["runs_per_cta"], f["ctas"]) == CV.plan(n, run_len), (shape, f)
        assert f["chunk"] == T and f["run_len"] == run_len
        assert f["load"] == ("vector" if strides[-1] == 1 and (len(shape) == 1 or strides[0] == shape[1]) else "strided"), (shape, f)


def test_malformed_compact_arguments_are_rejected():
    from ramba_b200 import _cabi

    lib = _cabi.load()
    P = 0x1000
    coords = onp.zeros(5, dtype=onp.int64)
    outs = (C.c_void_p * 5)(*([P] * 5))

    def count(view=None, dtype=4, run_len=6, counts=P):
        v = view if view is not None else _view([4, 6], [6, 1])
        return lib.rb200_compact_count(C.byref(v), dtype, run_len, counts, None), lib.rb200_last_error().decode()

    def compact(view=None, dtype=4, run_len=6, counts=P, form=0, values=None, origin=True, out=True):
        v = view if view is not None else _view([4, 6], [6, 1])
        vals = values if values is not None else _view([4, 6], [6, 1], eb=8)
        rc = lib.rb200_compact(C.byref(v), dtype, run_len, counts, P, P, form, C.byref(vals), coords.ctypes.data if origin else None,
                               coords.ctypes.data, outs if out else None, None)
        return rc, lib.rb200_last_error().decode()

    assert "bad condition dtype" in count(dtype=10)[1]
    assert "elem_bytes does not match" in count(dtype=0)[1]
    assert "run_len" in count(run_len=5)[1]
    assert "run_len" in count(run_len=0)[1]
    assert "null counts" in count(counts=None)[1]
    assert "null view base pointer" in count(view=_view([4, 6], [6, 1], base=0))[1]
    assert "outside its allocation" in count(view=_view([4, 6], [6, 1], bounds=(P, P + 20)))[1]
    assert "bad form" in compact(form=3)[1]
    assert "differ in shape" in compact(values=_view([4, 5], [5, 1], eb=8))[1]
    assert "compact values" in compact(values=_view([4, 6], [6, 1], eb=3))[1]
    assert "null origin" in compact(form=1, origin=False)[1]
    assert "null counts" in compact(counts=None)[1]
    assert "null out" in compact(out=False)[1]
    assert lib.rb200_describe_compact_plan(C.byref(_view([4, 6], [6, 1])), 7) is None
    import torch

    if not torch.cuda.is_available():
        assert "no usable CUDA device" in count()[1]
        assert "no usable CUDA device" in compact(form=2)[1]


def test_header_and_exports_agree():
    from ramba_b200 import _cabi

    head = open(os.path.join(HERE, "..", "include", "ramba_b200.h")).read()
    for name in ("rb200_compact_count", "rb200_compact", "rb200_describe_compact_plan"):
        assert name in _cabi.EXPORTS and re.search(r"\b%s\(" % name, head), name
    assert "#define RB200_COMPACT_CHUNK %d" % _cabi.COMPACT_CHUNK in head and _cabi.COMPACT_CHUNK == T
    assert "#define RB200_ABI_VERSION 7" in head


def test_compact_kernels_do_not_spill():
    """ptxas -v of rb200_compact.cu (written by the build): no kernel spills to local memory."""
    log = os.path.join(HERE, "..", "ramba_b200", "csrc", "build", "rb200_compact.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("library not built here")
    text = open(log).read()
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert spills and all(a == "0" and b == "0" for a, b in spills), spills
    assert text.count("Compiling entry function") == len(spills)


# ---- multi-rank over gloo -----------------------------------------------------------------------------------------------
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
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_compact_worker.py"), out, mode], env=env,
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


def _expected_programs():
    npns = types.SimpleNamespace(fromarray=onp.asarray, broadcast_to=onp.broadcast_to)
    out = {}
    for name, cond, vals in CW.programs():
        c = onp.asarray(cond(npns))
        for i, e in enumerate(onp.nonzero(c)):
            out["%s.nonzero.%d" % (name, i)] = e
        out["%s.flatnonzero.0" % name] = onp.flatnonzero(c)
        if vals is not None:
            out["%s.extract.0" % name] = onp.extract(c, onp.asarray(vals(npns)))
    return out


def _check_worlds(worlds):
    exp = _expected_programs()
    moved = False
    for w, res in worlds.items():
        assert set(k for k in res if not k.endswith(".counters")) == set(exp), w
        for k, e in exp.items():
            assert res[k].dtype == e.dtype and onp.array_equal(_bits(res[k]), _bits(e)), (w, k, res[k], e)
            assert onp.array_equal(_bits(res[k]), _bits(worlds[1][k])), (w, k)
        for k, c in res.items():
            if not k.endswith(".counters"):
                continue
            n_coll, n_p2p, n_bytes = (int(x) for x in c)
            if w == 1:
                assert n_coll == 0 and n_p2p == 0 and n_bytes == 0, (w, k, c)
            elif not k.startswith("bcast."):  # (a broadcast condition is copied first)
                assert n_coll == 1 and n_p2p <= 1, (w, k, c)
                moved |= n_p2p == 1
    assert moved


@pytest.fixture(scope="module")
def compact_worlds(tmp_path_factory):
    d = tmp_path_factory.mktemp("compact_worlds")
    return {w: _run_world(w, str(d / ("w%d.npz" % w))) for w in (1, 2, 3, 4, 8)}


@pytest.mark.timeout(1800)
def test_multirank_matches_one_rank_and_numpy(compact_worlds):
    _check_worlds(compact_worlds)


# ---- GPU ----------------------------------------------------------------------------------------------------------------
_CODE = {onp.dtype(onp.float64): 0, onp.dtype(onp.float32): 1, onp.dtype(onp.int64): 2, onp.dtype(onp.int32): 3, onp.dtype(onp.bool_): 4,
         onp.dtype(onp.uint8): 5, onp.dtype(onp.int8): 6, onp.dtype(onp.int16): 7, onp.dtype(onp.uint16): 8, onp.dtype(onp.uint32): 9}


def _gpu_vs_vm(shape, strides, run_len, dt, density=0.5, pad=16, seed=0, host=None):
    """One view of device memory through rb200_compact_count, the scan and rb200_compact in every form, against the
    restatement on the same bytes."""
    import torch

    from ramba_b200 import _cabi
    from ramba_b200.runtime import torch_dtype

    dev = torch.device("cuda", 0)
    lo = sum(min(0, (s - 1) * st) for s, st in zip(shape, strides))
    hi = sum(max(0, (s - 1) * st) for s, st in zip(shape, strides))
    nmem = hi - lo + 1 + 2 * pad
    if host is None:
        host = _data((nmem,), dt, seed, density)
    eb = host.dtype.itemsize
    d_mem = torch.from_numpy(host.view(onp.uint8).copy()).to(dev)
    base_off = (pad - lo) * eb
    view = _cabi.index_view(d_mem.data_ptr() + base_off, shape, strides, eb, (d_mem.data_ptr(), d_mem.data_ptr() + nmem * eb))
    h_view = _cabi.index_view(host.ctypes.data + base_off, shape, strides, eb)
    n = int(onp.prod(shape))
    n_runs, cpr = CV.plan(n, run_len)[:2]
    code = _CODE[host.dtype]
    counts = torch.zeros(n_runs * cpr, dtype=torch.int64, device=dev)
    _cabi.compact_count(view, code, run_len, counts.data_ptr())
    h_counts = onp.zeros(n_runs * cpr, dtype=onp.int64)
    CV.compact_count(h_view, code, run_len, h_counts.ctypes.data)
    assert counts.cpu().numpy().tolist() == h_counts.tolist(), (shape, strides, run_len, dt)
    incl = counts
    if cpr > 1:
        incl = torch.empty_like(counts)
        scratch = torch.empty(_cabi.cumulative_scratch_bytes(1, cpr, n_runs), dtype=torch.uint8, device=dev)
        _cabi.cumulative(counts.data_ptr(), incl.data_ptr(), 2, 1, cpr, n_runs, 0, None, None, scratch.data_ptr())
    h_incl = CV.inclusive(h_counts, n_runs)
    assert incl.cpu().numpy().tolist() == h_incl.tolist()
    tot = h_incl[(cpr - 1) * n_runs:]
    bases = onp.ascontiguousarray(onp.cumsum(tot) - tot + 3 * onp.arange(n_runs), dtype=onp.int64)  # gaps: bases are taken as given
    top = int(bases[-1] + tot[-1]) + 8
    d_base = torch.from_numpy(bases.copy()).to(dev)
    origin, gshape = [2] * len(shape), [s + 4 for s in shape]
    gstride = [int(onp.prod(gshape[d + 1:])) for d in range(len(shape))]
    vdt = {1: onp.uint8, 2: onp.int16, 4: onp.float32, 8: onp.float64}[eb]
    vals = _data((n,), vdt, seed + 1, 1.0).reshape(shape)
    d_vals = torch.from_numpy(vals.copy()).to(dev)
    vview = _cabi.index_view(d_vals.data_ptr(), shape, _cabi_strides(shape), vals.itemsize)
    hvview = _cabi.index_view(vals.ctypes.data, shape, _cabi_strides(shape), vals.itemsize)
    for form, k, odt in ((CV.VALUES, 1, vals.dtype), (CV.FLAT, 1, onp.int64), (CV.COORDS, len(shape), onp.int64)):
        d_out = [torch.full((top,), 77, dtype=torch_dtype(odt), device=dev) for _ in range(k)]
        h_out = [onp.full(top, 77, dtype=odt) for _ in range(k)]
        _cabi.compact(view, code, run_len, counts.data_ptr(), incl.data_ptr(), d_base.data_ptr(), form, vview if form == CV.VALUES else None,
                      origin, gstride, [t.data_ptr() for t in d_out])
        CV.compact(h_view, code, run_len, h_counts.ctypes.data, h_incl.ctypes.data, bases.ctypes.data, form,
                   hvview if form == CV.VALUES else None, origin, gstride, [a.ctypes.data for a in h_out])
        torch.cuda.synchronize()
        for t, a in zip(d_out, h_out):
            assert onp.array_equal(_bits(t.cpu().numpy()), _bits(a)), (shape, strides, run_len, dt, form)


def _cabi_strides(shape):
    return [int(onp.prod(shape[d + 1:])) for d in range(len(shape))]


@pytest.mark.gpu
def test_cuda_kernels_match_the_restatement():
    layouts = [  # (shape, strides, run_len)
        ([100003], [1], 100003),              # one long run, vector loads, ragged tail
        ([37, 301], [301, 1], 37 * 301),
        ([37, 301], [1, 37], 37 * 301),       # transposed: strided loads
        ([40, 90], [-90, 3], 40 * 90),        # reversed rows, stepped
        ([40, 9000], [9000, 1], 9000),        # runs of 3 chunks
        ([500, 31], [31, 1], 31),             # short runs, many per CTA
        ([4096, 1], [1, 1], 1),               # runs of one element
        ([6, 4, 33], [132, 33, 1], 33),
        ([5, 6, 7, 8], [336, 56, 8, 1], 56),
    ]
    for shape, strides, run_len in layouts:
        for dt in DTYPES:
            for density in (0.0, 0.01, 0.5, 1.0):
                _gpu_vs_vm(shape, strides, run_len, dt, density)


@pytest.mark.gpu
def test_cuda_chunk_edges():
    for dt in (onp.bool_, onp.float64):
        for n in (T - 1, T, T + 1, 2 * T - 1, 2 * T + 1):
            for run_len in (n, 1, 31, 32):
                if n % run_len == 0:
                    _gpu_vs_vm([n], [1], run_len, dt, 0.5, seed=n)
        for at in (0, T - 1, T, T + 1):  # a single selected element at a chunk edge, misaligned starts
            x = onp.zeros(3 * T + 40, dtype=dt)
            x[16 + 3 + at] = 1
            _gpu_vs_vm([3 * T], [1], 3 * T, dt, host=x, pad=16 + 3)


@pytest.mark.gpu
def test_cuda_extract_past_2_to_the_31():
    """extract on 2^31 + 5 uint8 elements at full density (64-bit positions and counts)."""
    import torch

    import ramba_b200 as rb
    from ramba_b200 import ramba
    from ramba_b200.runtime import RT

    if torch.cuda.get_device_properties(0).total_memory < (24 << 30):
        pytest.skip("needs 24 GB")
    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()
    n = (1 << 31) + 5
    A = rb.ones(n, dtype=onp.uint8)
    V = rb.arange(n).astype(onp.uint8)
    rb.sync()
    out = rb.extract(A, V)
    assert out.shape == (n,)
    sh = RT.shards[out.gid].buf
    for at in (0, 255, (1 << 31) - 1, 1 << 31, n - 1):
        assert int(sh[at]) == at % 256, at
    del out, sh, A, V
    RT.reset()
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_cuda_numpy_cases(gpu_engine):
    import ramba_b200 as rb

    _check_dtypes_and_ranks(rb)
    _check_views(rb)
    _check_densities_and_edges(rb)
    _check_pending_and_writes(rb)
    _check_errors_and_dispatch(rb)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_cuda_world2_over_nccl(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    one = _run_world(1, str(tmp_path / "w1.npz"), "cuda")
    two = _run_world(2, str(tmp_path / "w2.npz"), "cuda")
    _check_worlds({1: one, 2: two})
