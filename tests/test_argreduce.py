"""argmax, argmin, nanargmax and nanargmin: first-occurrence index reductions over every axis or along one.

CPU: the engine through the NumPy restatement of the kernel (_argred_vm) against NumPy with == for every stored dtype,
0-d to 4-d, every axis, keepdims, view kinds, ties, infinities, signed zeros and NaN placements; the errors; gloo worlds
2, 3, 4 and 8 against world 1 with the transfer counters; the restatement against a per-element brute force; the plan
and the argument checks of the C-ABI; no spills.
GPU: rb200_arg_reduce against the restatement in every form and dtype, past 2^31 elements and at CTA tile boundaries;
the NumPy cases through the CUDA library; world 2 over NCCL where two GPUs exist."""
import ctypes as C
import os
import re
import socket
import subprocess
import sys

import numpy as onp
import pytest

import _argred_vm as AV
import _argred_worker as AW

HERE = os.path.dirname(os.path.abspath(__file__))
FUNCS = AW.FUNCS
AV.extend_oracle_backend()  # (also for the oracle stand-in of the -m gpu tests under RB200_DRY_GPU_TESTS)
DTYPES = (onp.float64, onp.float32, onp.int64, onp.int32, onp.bool_, onp.uint8, onp.int8, onp.int16, onp.uint16, onp.uint32)


@pytest.fixture
def arg_engine():
    import _oracle_backend
    from ramba_b200 import ramba
    from ramba_b200.runtime import RT

    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()
    _oracle_backend.install()
    yield
    ramba.deferred_op.ramba_deferred_ops = None
    RT.reset()


def _data(shape, dtype, seed):
    """Few distinct values (many ties); floats get -0.0, +-inf and NaN."""
    r = onp.random.default_rng(seed)
    x = r.integers(-3, 4, size=shape)
    if onp.dtype(dtype) == onp.bool_:
        return (x > 0)
    if onp.dtype(dtype).kind == "u":
        return (x + 3).astype(dtype)
    x = x.astype(dtype)
    if x.dtype.kind == "f" and x.size > 4:
        f = x.reshape(-1)
        f[r.integers(0, f.size, 3)] = -0.0
        f[r.integers(0, f.size, 2)] = onp.inf
        f[r.integers(0, f.size, 2)] = -onp.inf
    return x


def _same(got, exp, what):
    if isinstance(exp, onp.ndarray) and exp.ndim:
        from ramba_b200 import ndarray

        assert isinstance(got, ndarray), what
        g = got.asarray()
        assert g.dtype == onp.int64 and g.shape == exp.shape and onp.array_equal(g, exp), (what, g, exp)
    else:
        assert isinstance(got, onp.int64) and got == exp, (what, got, exp)


def _check(rb, hv, A, funcs=FUNCS, axes=None):
    axes = [None] + list(range(-hv.ndim, hv.ndim)) if axes is None else axes
    for f in funcs:
        if f.startswith("nan") and hv.dtype.kind == "f" and onp.isnan(hv).all() and hv.size:
            continue
        for ax in axes:
            for kd in (False, True):
                try:
                    exp = getattr(onp, f)(hv, axis=ax, keepdims=kd)
                except ValueError:
                    with pytest.raises(ValueError):
                        getattr(rb, f)(A, axis=ax, keepdims=kd)
                    continue
                _same(getattr(rb, f)(A, axis=ax, keepdims=kd), exp, (f, ax, kd, hv.dtype, hv.shape))


SHAPES = [(), (7,), (5, 9), (3, 4, 5), (2, 3, 4, 5)]


def _check_dtypes_and_ranks(rb, dtypes=DTYPES):
    for dt in dtypes:
        for i, shape in enumerate(SHAPES):
            x = _data(shape, dt, i)
            _check(rb, x, rb.fromarray(x) if shape else rb.array(x))


def test_every_dtype_rank_axis_and_keepdims(arg_engine):
    import ramba_b200 as rb

    _check_dtypes_and_ranks(rb)


VIEWS = [
    ("sliced", (9, 50), lambda x: x[1:8, 3:43]),
    ("stepped", (9, 90), lambda x: x[::2, ::3]),
    ("reversed", (5, 40), lambda x: x[::-1, ::-1]),
    ("transposed", (40, 7), lambda x: x.T),
    ("transposed3", (4, 6, 5), lambda x: x.transpose(2, 0, 1) if isinstance(x, onp.ndarray) else x.transpose(2, 0, 1)),
    ("broadcast", (1, 40), lambda x: onp.broadcast_to(x, (4, 40)) if isinstance(x, onp.ndarray) else x.broadcast_to((4, 40))),
    ("lazy", (6, 40), lambda x: x * 2 - 1),
]


def _check_views(rb, dtypes=(onp.float64, onp.float32, onp.int64, onp.int32, onp.int16)):
    for name, shape, view in VIEWS:
        for dt in dtypes:
            x = _data(shape, dt, 3)
            _check(rb, onp.asarray(view(x)), view(rb.fromarray(x)))
    x = _data((12, 10), onp.float64, 4)  # a padded shard
    _check(rb, x[2:9, 1:8], rb.fromarray(x, local_border=2)[2:9, 1:8])


def test_views_and_lazy_sources(arg_engine):
    import ramba_b200 as rb

    _check_views(rb)


def _nan_cases():
    n = onp.nan
    yield onp.array([n, 1.0, 5.0, 5.0])                     # NaN first
    yield onp.array([1.0, 5.0, n, 7.0, n])                  # middle
    yield onp.array([1.0, 5.0, 5.0, 0.5, n])                # last
    yield onp.array([-0.0, 0.0, -0.0, 0.0])                 # signed zeros tie
    yield onp.array([onp.inf, -onp.inf, onp.inf, -onp.inf])
    yield onp.array([[n, n, 1.0], [n, n, n], [2.0, n, 2.0]])  # an all-NaN row and column
    yield onp.array([[n, n], [n, n]], dtype=onp.float32)
    yield onp.full((3, 4), 2.5, dtype=onp.float32)
    yield onp.array([onp.iinfo(onp.int64).min, onp.iinfo(onp.int64).max, onp.iinfo(onp.int64).min, onp.iinfo(onp.int64).max])


def _check_nan_and_ties(rb):
    for x in _nan_cases():
        _check(rb, x, rb.fromarray(x))
        for f in FUNCS:
            try:
                getattr(onp, f)(x)
            except ValueError as e:
                with pytest.raises(ValueError, match=re.escape(str(e))):
                    getattr(rb, f)(rb.fromarray(x))
    x = onp.array([[onp.nan, 1.0], [onp.nan, onp.nan]])
    with pytest.raises(ValueError, match="All-NaN slice encountered"):
        rb.nanargmin(rb.fromarray(x), axis=1)
    with pytest.raises(ValueError, match="All-NaN slice encountered"):
        rb.nanargmax(rb.fromarray(x[1]))


def test_nan_ties_and_signed_zeros(arg_engine):
    import ramba_b200 as rb

    _check_nan_and_ties(rb)


def _check_errors(rb):
    A = rb.fromarray(onp.arange(12.0).reshape(3, 4))
    with pytest.raises(TypeError):
        rb.argmax(A, axis=(0,))
    with pytest.raises(TypeError):
        A.argmin(axis=1.0)
    with pytest.raises(onp.exceptions.AxisError):
        A.argmax(axis=2)
    with pytest.raises(onp.exceptions.AxisError):
        rb.nanargmin(A, axis=-3)
    with pytest.raises(NotImplementedError):
        A.argmax(out=onp.zeros(4, dtype=onp.int64))
    with pytest.raises(NotImplementedError):
        A[A > 3.0].argmax()
    for shape, ax, f in (((0, 3), 0, "argmax"), ((0, 0), 0, "argmin"), ((0,), None, "nanargmax"), ((2, 0), None, "argmin")):
        with pytest.raises(ValueError, match="attempt to get %s of an empty sequence" % f.replace("nan", "")):
            getattr(rb, f)(rb.zeros(shape), axis=ax)
    e = rb.zeros((3, 0)).argmax(axis=0)
    assert e.shape == (0,) and e.asarray().dtype == onp.int64
    assert rb.zeros((3, 0)).argmin(axis=0, keepdims=True).shape == (1, 0)
    # NumPy's functions dispatch here
    x = _data((6, 7), onp.float64, 9)
    X = rb.fromarray(x)
    assert onp.argmax(X) == onp.argmax(x) and isinstance(onp.argmax(X), onp.int64)
    _same(onp.nanargmin(X, axis=1), onp.nanargmin(x, axis=1), "np.nanargmin")
    _same(rb.nanargmin(X, axis=1), onp.nanargmin(x, axis=1), "rb.nanargmin")


def test_errors_and_dispatch(arg_engine):
    import ramba_b200 as rb

    _check_errors(rb)


# ---- the restatement against a per-element brute force ----------------------------------------------------------------
def _brute(x, axis, op, origin, gstride):
    def better(k, i, k2, i2):
        return k2 > k or (k2 == k and i2 < i)

    nan_variant = op in (AV.ARG_NANMAX, AV.ARG_NANMIN)

    def key(v):
        if x.dtype.kind == "f":
            if onp.isnan(v):
                if nan_variant:
                    return None
                return AV.NO_INDEX if op == AV.ARG_MAX else ~AV.KEY_MIN
            v = abs(v) if v == 0 else v
            b = int(onp.array(v, x.dtype).view(onp.int64 if x.dtype.itemsize == 8 else onp.int32))
            k = b if b >= 0 else b ^ AV.NO_INDEX
        else:
            k = int(v)
        return ~k if op in (AV.ARG_MIN, AV.ARG_NANMIN) else k

    if axis == AV.ALL_AXES:
        groups = {(): list(onp.ndindex(x.shape))}
    else:
        groups = {}
        for c in onp.ndindex(x.shape):
            groups.setdefault(c[:axis] + c[axis + 1:], []).append(c)
    out_shape = () if axis == AV.ALL_AXES else x.shape[:axis] + x.shape[axis + 1:]
    idx = onp.full(out_shape, AV.NO_INDEX, dtype=onp.int64)
    kk = onp.full(out_shape, AV.KEY_MIN, dtype=onp.int64)
    for o, cs in groups.items():
        bk, bi = AV.KEY_MIN, AV.NO_INDEX
        for c in cs:
            k = key(x[c])
            if k is None:
                continue
            g = sum((c[d] + origin[d]) * gstride[d] for d in range(x.ndim)) if axis == AV.ALL_AXES else c[axis] + origin[axis]
            if better(bk, bi, k, g):
                bk, bi = k, g
        idx[o], kk[o] = bi, bk
    return idx, kk


def test_restatement_against_brute_force():
    rng = onp.random.default_rng(0)
    for trial in range(40):
        shape = [int(rng.integers(1, 5)) for _ in range(int(rng.integers(1, 4)))]
        dt = [onp.float64, onp.float32, onp.int64, onp.int32][trial % 4]
        x = rng.integers(-2, 3, size=shape).astype(dt)
        if x.dtype.kind == "f":
            f = x.reshape(-1)
            f[rng.random(f.size) < 0.25] = onp.nan
            f[rng.random(f.size) < 0.2] = -0.0
        gshape = [s + int(rng.integers(0, 4)) for s in shape]
        origin = [int(rng.integers(0, g - s + 1)) for g, s in zip(gshape, shape)]
        gstride = [int(onp.prod(gshape[d + 1:])) for d in range(len(shape))]
        for axis in [AV.ALL_AXES] + list(range(len(shape))):
            for op in range(4):
                got = AV.reduce(x, axis, op, origin, gstride)
                exp = _brute(x, axis, op, origin, gstride)
                assert onp.array_equal(got[0], exp[0]) and onp.array_equal(got[1], exp[1]), (trial, axis, op, x, got, exp)


# ---- the C-ABI ---------------------------------------------------------------------------------------------------------
def _view(shape, strides, eb=8, base=0x1000, bounds=None):
    from ramba_b200 import _cabi

    return _cabi.index_view(base, shape, strides, eb, bounds)


PLAN_CASES = [  # (shape, strides, axis, form, split?)
    ([65536, 4096], [4096, 1], 1, "row", False),
    ([65536, 4096], [4096, 1], 0, "column", True),
    ([1 << 30], [1], -1, "global", True),
    ([65536, 4096], [4096, 1], -1, "global", True),
    ([300, 70], [1, 300], 1, "general", False),        # transposed
    ([30, 90], [-90, 2], 1, "general", False),         # reversed rows, stepped axis
    ([20, 31, 7], [217, 7, 1], 1, "general", False),   # middle axis, short inner run
    ([5, 100000], [100000, 1], 1, "row", True),        # too few rows: the axis is split
    ([40, 50], [0, 1], 1, "row", False),               # broadcast rows
    ([3000, 64], [64, 1], 0, "column", True),
    ([7, 9], [9, 1], -1, "global", False),
]


def test_describe_arg_plan_matches_the_restatement():
    from ramba_b200 import _cabi

    for shape, strides, axis, form, split in PLAN_CASES:
        f = _cabi.group_plan_fields(_cabi.describe_arg_plan(_view(shape, strides), axis))
        assert f["form"] == form and (f["split"] > 1) == split, (shape, strides, axis, f)
        assert AV.plan(shape, strides, axis) == (form, f["chunk"], f["split"]), (shape, f)
        assert f["scratch"] == (16 * f["split"] * f["outputs"] if f["split"] > 1 else 0)
        assert _cabi.arg_reduce_scratch_bytes(_view(shape, strides), axis) == f["scratch"]


def test_malformed_arg_arguments_are_rejected():
    from ramba_b200 import _cabi

    lib = _cabi.load()
    P = 0x1000
    coords = onp.zeros(5, dtype=onp.int64)

    def call(view=None, dtype=0, axis=1, op=0, origin=True, out_idx=P, out_key=P, scratch=P):
        v = view if view is not None else _view([4, 6], [6, 1])
        rc = lib.rb200_arg_reduce(C.byref(v), dtype, axis, op, coords.ctypes.data if origin else None, coords.ctypes.data, out_idx, out_key, scratch,
                                  None)
        return rc, lib.rb200_last_error().decode()

    assert "bad op" in call(op=4)[1]
    assert "bad op" in call(op=-1)[1]
    assert "source dtype" in call(dtype=4)[1]
    assert "elem_bytes does not match" in call(dtype=1)[1]
    assert "axis out of range" in call(axis=2)[1]
    assert "axis out of range" in call(axis=-2)[1]
    assert "null out" in call(out_idx=None)[1]
    assert "null out" in call(out_key=None)[1]
    assert "null origin" in call(origin=False)[1]
    assert "null view base pointer" in call(view=_view([4, 6], [6, 1], base=0))[1]
    assert "elem_bytes" in call(view=_view([4, 6], [6, 1], eb=3))[1]
    assert "outside its allocation" in call(view=_view([4, 6], [6, 1], bounds=(P, P + 8 * 20)))[1]
    assert "null scratch" in call(view=_view([1 << 20], [1]), axis=-1, scratch=None)[1]
    assert lib.rb200_describe_arg_plan(C.byref(_view([4, 6], [6, 1])), 5) is None
    assert lib.rb200_arg_reduce_scratch_bytes(C.byref(_view([4, 6], [6, 1])), 3) < 0
    import torch

    if not torch.cuda.is_available():
        assert "no usable CUDA device" in call()[1]


def test_arg_kernels_do_not_spill():
    """ptxas -v of rb200_argred.cu (written by the build): no kernel spills to local memory."""
    log = os.path.join(HERE, "..", "ramba_b200", "csrc", "build", "rb200_argred.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("library not built here")
    text = open(log).read()
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert spills and all(a == "0" and b == "0" for a, b in spills), spills
    assert text.count("Compiling entry function") == len(spills)


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
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_argred_worker.py"), out, mode], env=env,
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
    import types

    class _NP(types.SimpleNamespace):
        pass

    npns = _NP(fromarray=onp.asarray)
    out = {}
    for name, build, axis in AW.programs():
        try:
            x = onp.asarray(build(npns))
        except AttributeError:  # .broadcast_to of the ramba spelling
            continue
        for f in FUNCS:
            out["%s.%s" % (name, f)] = getattr(onp, f)(x, axis=axis)
    return out


def _check_worlds(worlds):
    base = worlds[1]
    exp = _expected_programs()
    cuts = set()
    for w, res in worlds.items():
        for k, v in res.items():
            if k.endswith(".counters"):
                continue
            assert onp.array_equal(v, base[k]), (w, k, v, base[k])
            if k in exp:
                assert onp.array_equal(v, exp[k]), (w, k, v, exp[k])
        for k, c in res.items():
            if not k.endswith(".counters"):
                continue
            f = k.split(".")[1]
            n_coll, n_bytes, cut, size, is_float = (int(x) for x in c)
            cuts.add((w > 1, bool(cut)))
            if w == 1:
                assert n_coll == 0 and n_bytes == 0, (w, k, c)
            elif cut:
                assert n_coll == 2 and n_bytes == 2 * 8 * size, (w, k, c)
            else:
                extra = 1 if f.startswith("nan") and is_float else 0  # the all-NaN check agrees across ranks
                assert n_coll == extra and n_bytes == 8 * extra, (w, k, c)
    assert (True, True) in cuts and (True, False) in cuts, cuts  # both layouts ran at several ranks


@pytest.fixture(scope="module")
def arg_worlds(tmp_path_factory):
    d = tmp_path_factory.mktemp("arg_worlds")
    return {w: _run_world(w, str(d / ("w%d.npz" % w))) for w in (1, 2, 3, 4, 8)}


@pytest.mark.timeout(1800)
def test_multirank_matches_one_rank_and_numpy(arg_worlds):
    _check_worlds(arg_worlds)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
_CODE = {onp.dtype(onp.float64): 0, onp.dtype(onp.float32): 1, onp.dtype(onp.int64): 2, onp.dtype(onp.int32): 3}


def _gpu_vs_vm(shape, strides, axis, dt, pad=16, seed=0, host=None):
    """One view of device memory through rb200_arg_reduce and the restatement: the same indices and keys for every op."""
    import torch

    from ramba_b200 import _cabi

    dev = torch.device("cuda", 0)
    rng = onp.random.default_rng(seed)
    lo = sum(min(0, (s - 1) * st) for s, st in zip(shape, strides))
    hi = sum(max(0, (s - 1) * st) for s, st in zip(shape, strides))
    nmem = hi - lo + 1 + 2 * pad
    if host is None:
        host = rng.integers(-40, 40, size=nmem).astype(dt)
        if onp.dtype(dt).kind == "f":
            host[rng.random(nmem) < 0.01] = onp.nan
            host[rng.random(nmem) < 0.01] = -0.0
    eb = onp.dtype(dt).itemsize
    d_mem = torch.from_numpy(host.copy()).to(dev)
    base_off = (pad - lo) * eb
    view = _cabi.index_view(d_mem.data_ptr() + base_off, shape, strides, eb, (d_mem.data_ptr(), d_mem.data_ptr() + nmem * eb))
    h_view = _cabi.index_view(host.ctypes.data + base_off, shape, strides, eb)
    gshape = [s + 3 for s in shape]
    origin = [1] * len(shape)
    gstride = [int(onp.prod(gshape[d + 1:])) for d in range(len(shape))]
    n_out = 1 if axis == AV.ALL_AXES else int(onp.prod(shape[:axis] + shape[axis + 1:]))
    scratch = torch.empty(max(_cabi.arg_reduce_scratch_bytes(view, axis), 1), dtype=torch.uint8, device=dev)
    form = _cabi.group_plan_fields(_cabi.describe_arg_plan(view, axis))
    o, g = _cabi.arg_coords(origin, gstride)
    for op in range(4):
        d_idx = torch.full((max(n_out, 1),), 7, dtype=torch.int64, device=dev)
        d_key = torch.full((max(n_out, 1),), 7, dtype=torch.int64, device=dev)
        _cabi.arg_reduce(view, _CODE[onp.dtype(dt)], axis, op, o, g, d_idx.data_ptr(), d_key.data_ptr(), scratch.data_ptr())
        h_idx = onp.zeros(max(n_out, 1), dtype=onp.int64)
        h_key = onp.zeros(max(n_out, 1), dtype=onp.int64)
        AV.arg_reduce(h_view, _CODE[onp.dtype(dt)], axis, op, origin, gstride, h_idx.ctypes.data, h_key.ctypes.data)
        torch.cuda.synchronize()
        assert d_idx.cpu().numpy()[:n_out].tolist() == h_idx[:n_out].tolist(), (shape, strides, axis, dt, op, form)
        assert d_key.cpu().numpy()[:n_out].tolist() == h_key[:n_out].tolist(), (shape, strides, axis, dt, op, form)
    return form["form"], form["split"] > 1


@pytest.mark.gpu
def test_cuda_kernel_matches_the_restatement_every_form():
    seen = set()
    layouts = [  # (shape, strides, axis)
        ([100003], [1], -1),               # global, one unit-stride run, ragged tail
        ([37, 301], [301, 1], -1),         # global, merged dims
        ([37, 301], [1, 37], -1),          # global, transposed: decoded walk
        ([40, 90], [-90, 3], -1),          # global, reversed rows, stepped
        ([1], [1], -1),
        ([37, 301], [301, 1], 1),          # row
        ([3, 50001], [50001, 1], 1),       # row, split (ragged)
        ([12, 40], [0, 1], 1),             # broadcast rows
        ([301, 70], [70, 1], 0),           # column
        ([5000, 33], [33, 1], 0),          # column, split
        ([60, 41], [1, 60], 1),            # transposed: general
        ([30, 90], [-90, 2], 1),           # general
        ([20, 31, 7], [217, 7, 1], 1),     # middle axis, short inner run: general
        ([5, 40, 3, 4], [480, 12, 4, 1], 1),
        ([4000, 3], [3, 1], 0),            # general, split
    ]
    for shape, strides, axis in layouts:
        for dt in (onp.float64, onp.float32, onp.int64, onp.int32):
            seen.add(_gpu_vs_vm(shape, strides, axis, dt))
    assert {f for f, _ in seen} == {"global", "row", "column", "general"}
    assert {f for f, s in seen if s} >= {"global", "row", "column", "general"}


@pytest.mark.gpu
def test_cuda_maxima_at_tile_boundaries():
    """A single maximum (and a tie right after it) at the edges of CTA chunks, vector loads and warps."""
    from ramba_b200 import _cabi

    n = 3 * 1056 * 4096 + 77
    chunk = _cabi.group_plan_fields(_cabi.describe_arg_plan(_view([n], [1]), -1))["chunk"]
    for dt in (onp.float64, onp.float32):
        for at in (0, 1, 3, 4, chunk - 1, chunk, chunk + 1, 2 * chunk - 2, n - 2, n - 1):
            x = onp.zeros(n + 32, dtype=dt)
            x[16 + at] = 5
            if at + 1 < n:
                x[16 + at + 1] = 5
            _gpu_vs_vm([n], [1], -1, dt, host=x)
    for at in (0, 31, 32, 1087, 1088, 50000):  # the split row form's chunk edges
        x = onp.zeros(3 * 50001 + 32, dtype=onp.float64)
        x[16 + 50001 + at] = 9
        _gpu_vs_vm([3, 50001], [50001, 1], 1, onp.float64, host=x)


@pytest.mark.gpu
def test_cuda_kernel_past_2_to_the_31():
    """One f32 view of more than 2^31 elements (64-bit indices): the maximum at the last element and at 2^31 + k."""
    import torch

    from ramba_b200 import _cabi

    if torch.cuda.get_device_properties(0).total_memory < (16 << 30):
        pytest.skip("needs 16 GB")
    rows, L = 65540, 32768  # 2^31 + 131072 elements
    n = rows * L
    dev = torch.device("cuda", 0)
    src = torch.zeros(n, dtype=torch.float32, device=dev)
    view = _cabi.index_view(src.data_ptr(), [rows, L], [L, 1], 4, (src.data_ptr(), src.data_ptr() + n * 4))
    o, g = _cabi.arg_coords([0, 0], [L, 1])
    idx = torch.zeros(rows, dtype=torch.int64, device=dev)
    key = torch.zeros(rows, dtype=torch.int64, device=dev)
    for at in (n - 1, (1 << 31) + 12345):
        src[at] = 3.0
        for axis in (-1, 1, 0):
            scratch = torch.empty(max(_cabi.arg_reduce_scratch_bytes(view, axis), 1), dtype=torch.uint8, device=dev)
            _cabi.arg_reduce(view, 1, axis, AV.ARG_MAX, o, g, idx.data_ptr(), key.data_ptr(), scratch.data_ptr())
            torch.cuda.synchronize()
            if axis == -1:
                assert int(idx[0]) == at, (axis, at)
            elif axis == 1:
                assert int(idx[at // L]) == at % L and int(idx[0]) == 0, (axis, at)
            else:
                assert int(idx[at % L]) == at // L, (axis, at)
            del scratch
        src[at] = 0.0
    del src
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_cuda_numpy_cases(gpu_engine):
    import ramba_b200 as rb

    _check_dtypes_and_ranks(rb)
    _check_views(rb)
    _check_nan_and_ties(rb)
    _check_errors(rb)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_cuda_world2_over_nccl(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    one = _run_world(1, str(tmp_path / "w1.npz"), "cuda")
    two = _run_world(2, str(tmp_path / "w2.npz"), "cuda")
    _check_worlds({1: one, 2: two})
