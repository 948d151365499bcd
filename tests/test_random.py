"""`ramba_b200.random`: counter-based Philox draws (RB200_OP_PHILOX, include/ramba_b200.h).

CPU: the block function against the CUDA toolkit's own Philox, the value contract pinned by literals, bit-identical
arrays over gloo at world sizes 1-4, fused and materialised draws agreeing, statistics, errors and plan selection.
GPU: the fill kernel and the general interpreter against the NumPy restatement of the contract (_philox_vm)."""
import os
import shutil
import socket
import subprocess
import sys

import numpy as onp
import pytest

import _philox_vm as P

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")


# ---------------------------------------------------------------------------------------------------------------------
# the generator
KAT = [  # Random123 known-answer vectors of Philox4x32-10: counter (4 words), key (2 words) -> 4 words
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]

_CURAND_MAIN = r"""
#define QUALIFIERS static inline __host__ __device__
#include <curand_philox4x32_x.h>
#include <stdio.h>
int main() {
  unsigned c0, c1, c2, c3, k0, k1;
  while (scanf("%u %u %u %u %u %u", &c0, &c1, &c2, &c3, &k0, &k1) == 6) {
    uint4 w = curand_Philox4x32_10(make_uint4(c0, c1, c2, c3), make_uint2(k0, k1));
    printf("%u %u %u %u\n", w.x, w.y, w.z, w.w);
  }
  return 0;
}
"""


def test_known_answer_vectors():
    for c, k, w in KAT:
        got = P.philox4x32_10(*c, *k)
        assert tuple(int(x) for x in got) == w


def test_block_function_matches_the_cuda_toolkit(tmp_path):
    """The oracle's Philox4x32-10 against curand's, compiled for the host, on the known-answer vectors and 10^4 seeded
    (counter, key) pairs."""
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("needs nvcc")
    src = tmp_path / "kat.cu"
    src.write_text(_CURAND_MAIN)
    exe = tmp_path / "kat"
    subprocess.check_call([nvcc, "-O1", "-o", str(exe), str(src)])
    rng = onp.random.default_rng(2024)
    words = rng.integers(0, 1 << 32, size=(10000, 6), dtype=onp.uint64)
    words[:3] = [list(c) + list(k) for c, k, _ in KAT]
    inp = "\n".join(" ".join(str(int(x)) for x in row) for row in words) + "\n"
    out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout
    ref = onp.array([[int(x) for x in line.split()] for line in out.strip().splitlines()], dtype=onp.uint64)
    got = onp.stack(P.philox4x32_10(*[words[:, q] for q in range(6)]), axis=1)
    assert ref.shape == (10000, 4)
    assert onp.array_equal(got, ref)
    assert [tuple(int(x) for x in ref[i]) for i in range(3)] == [w for _, _, w in KAT]


def test_key_derivation_is_pinned():
    from ramba_b200 import random as R

    assert R.splitmix64(0) == 0xE220A8397B1DCDAF
    assert R.draw_key(0, 0) == 0xA706DD2F4D197E6F
    assert R.draw_key(12345, 7) == 0xFBDF4C68FA8AFDEC


# ---------------------------------------------------------------------------------------------------------------------
# engine on the CPU: op lists through the NumPy oracle extended by PHILOX
@pytest.fixture
def engine(oracle_engine):
    import _oracle_backend

    del _oracle_backend.PLANS[:]
    return _oracle_backend.PLANS


SEED0 = {
    "u64": [float.fromhex(h) for h in ("0x1.f1b82461e36c8p-1", "0x1.8c91904304bb2p-2", "0x1.3dbff576666f4p-3", "0x1.b0b595744db6ap-2",
                                       "0x1.c61a6a12ce19dp-1", "0x1.cc9f01d68e610p-4", "0x1.9ff8d3ed7bfd4p-3", "0x1.aed788e54d3c6p-2")],
    "u32": [float.fromhex(h) for h in ("0x1.a892780000000p-2", "0x1.baa3f40000000p-1", "0x1.1ea3c20000000p-1", "0x1.3557d60000000p-1",
                                       "0x1.e311140000000p-1", "0x1.22f6680000000p-1", "0x1.d9f5080000000p-2", "0x1.4e4ee00000000p-5")],
    "n64": [-0.13636118714161757, 2.280864625777644, 0.07442996706890789, -0.3142273304968091, 0.18352533033365623,
            -1.1060412894662668, 0.007835464472665142, -0.34453706300155373],
    "int": [412, 765, 995, 52, 431, 791, 979, 326],
}


def test_seed0_values_are_pinned(engine):
    import ramba_b200 as rb

    rb.random.seed(0)
    u64 = rb.random.random(8).asarray()
    u32 = rb.random.random(8, dtype=onp.float32).asarray()
    n64 = rb.random.randn(8).asarray()
    i64 = rb.random.randint(0, 1000, 8).asarray()
    assert u64.dtype == onp.float64 and u32.dtype == onp.float32 and n64.dtype == onp.float64 and i64.dtype == onp.int64
    assert u64.tolist() == SEED0["u64"]
    assert u32.astype(onp.float64).tolist() == SEED0["u32"]
    assert onp.allclose(n64, SEED0["n64"], rtol=0, atol=1e-13)
    assert i64.tolist() == SEED0["int"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run_world(world, out, extra_env=None):
    port = _free_port()
    procs = []
    for r in range(world):
        env = dict(os.environ)
        env.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r), "MASTER_ADDR": "127.0.0.1",
                    "MASTER_PORT": str(port), "OMP_NUM_THREADS": "1"})
        env.update(extra_env or {})
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_random_worker.py"), out], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=240)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, o))
    for rc, o in outs:
        assert rc == 0, o[-3000:]
    return dict(onp.load(out))


@pytest.fixture(scope="module")
def worlds(tmp_path_factory):
    d = tmp_path_factory.mktemp("worlds")
    return {w: _run_world(w, str(d / ("w%d.npz" % w))) for w in (1, 2, 3, 4)}


@pytest.mark.timeout(600)
def test_draws_do_not_depend_on_the_number_of_ranks(worlds):
    base = worlds[1]
    for w in (2, 3, 4):
        assert set(worlds[w]) == set(base)
        for k, v in base.items():
            assert v.dtype == worlds[w][k].dtype, (w, k)
            if ".fsum" in k:  # float reductions: same terms, summed in another order
                assert onp.allclose(v, worlds[w][k], rtol=1e-12, atol=0), (w, k)
            else:
                assert onp.array_equal(v, worlds[w][k]), (w, k)
    # the second run of every program (flush scripts replayed) gives the first run's arrays
    for k, v in base.items():
        if k.endswith(".0"):
            assert onp.array_equal(v, base[k[:-1] + "1"]), k


@pytest.mark.timeout(600)
def test_multirank_draws_follow_the_contract(worlds):
    from ramba_b200 import random as R

    r = worlds[1]
    assert onp.array_equal(r["plain.u1.0"], P.draw(onp.arange(1001), R.draw_key(7, 0), P.UNIFORM64))
    assert onp.array_equal(r["plain.small.0"], P.draw(onp.arange(5), R.draw_key(7, 1), P.UNIFORM64))
    lin = onp.arange(37 * 53).reshape(37, 53)
    assert onp.array_equal(r["plain.u32.0"], P.draw(lin, R.draw_key(7, 2), P.UNIFORM32))
    lin = onp.arange(64 * 33).reshape(64, 33)
    assert onp.array_equal(r["plain.n2.0"], 2.0 + 3.0 * P.draw(lin, R.draw_key(7, 3), P.NORMAL64))
    lin = onp.arange(11 * 7 * 5).reshape(11, 7, 5)
    assert onp.array_equal(r["plain.i3.0"], 3 + P.draw(lin, R.draw_key(7, 4), P.INTEGER, 14))
    a = onp.zeros((40, 30))
    a[5:25, 3:13] = P.draw(onp.arange(200).reshape(20, 10), R.draw_key(8, 0), P.UNIFORM64)
    assert onp.array_equal(r["views.a.0"], a)
    b = onp.zeros((30, 40))
    b.T[:, :] = P.draw(onp.arange(1200).reshape(40, 30), R.draw_key(8, 1), P.NORMAL64)
    assert onp.array_equal(r["views.b.0"], b)
    x = P.draw(onp.arange(5000), R.draw_key(9, 0), P.UNIFORM64)
    y = P.draw(onp.arange(5000), R.draw_key(9, 1), P.UNIFORM64)
    assert int(r["fused.inside.0"]) == int(((x * x + y * y) < 1.0).sum())
    z = P.draw(onp.arange(3000).reshape(60, 50), R.draw_key(9, 2), P.NORMAL64)
    assert onp.array_equal(r["fused.colcount.0"], ((z * 2.0 + 1.0) > 0.0).sum(axis=0))


def _fused_and_kept(rb):
    """The same draws as a kept array and as a dead temporary folded into its consumer."""
    rb.random.seed(21)
    x = rb.random.normal(1.0, 2.0, (300, 7))
    kept = (x * 3.0 - 1.0).asarray()
    xs = x.asarray()
    rb.random.seed(21)
    folded = (rb.random.normal(1.0, 2.0, (300, 7)) * 3.0 - 1.0).asarray()
    rb.random.seed(21)
    s_fold = float((rb.random.normal(1.0, 2.0, (300, 7)) * 3.0 - 1.0).sum())
    return xs, kept, folded, s_fold


@pytest.mark.parametrize("mode", ["default", "no_dag", "verify_lower", "verify_plan"])
def test_fused_and_materialised_draws_agree(engine, monkeypatch, mode):
    import ramba_b200 as rb
    from ramba_b200 import flush, ramba, runtime

    if mode == "no_dag":
        monkeypatch.setattr(ramba, "NO_DAG", True)
    elif mode == "verify_lower":
        monkeypatch.setattr(ramba, "_VERIFY_LOWER_CACHE", True)
    elif mode == "verify_plan":
        monkeypatch.setattr(flush, "_VERIFY_PLAN_CACHE", True)
        monkeypatch.setattr(runtime, "_VERIFY_PLAN_CACHE", True)
    for _ in range(2):  # the second round hits the memos
        xs, kept, folded, s_fold = _fused_and_kept(rb)
        assert onp.array_equal(kept, xs * 3.0 - 1.0)
        assert onp.array_equal(kept, folded)
        assert abs(s_fold - float((xs * 3.0 - 1.0).sum())) <= 1e-12 * abs(s_fold)  # (a sum in another order)


def test_a_pruned_draw_still_advances_the_counter(engine):
    import ramba_b200 as rb

    rb.random.seed(5)
    rb.random.rand(10)
    second = rb.random.rand(10).asarray()
    rb.random.seed(5)
    a = rb.random.rand(10)
    del a  # never computed
    b = rb.random.rand(10).asarray()
    assert onp.array_equal(b, second)


def test_statistics(engine):
    import ramba_b200 as rb

    n = 10 ** 6
    rb.random.seed(123)
    u = rb.random.random(n).asarray()
    f = rb.random.random(n, dtype=onp.float32).asarray().astype(onp.float64)
    z = rb.random.randn(n).asarray()
    for x in (u, f):
        assert abs(x.mean() - 0.5) < 5 * (1 / 12) ** 0.5 / n ** 0.5
        assert abs(x.var() - 1 / 12) < 5 * (1 / 180) ** 0.5 / n ** 0.5
        assert x.min() >= 0.0 and x.max() < 1.0
    assert abs(z.mean()) < 5 / n ** 0.5 and abs(z.var() - 1.0) < 5 * 2 ** 0.5 / n ** 0.5
    k = rb.random.randint(-3, 17, n).asarray()
    assert k.min() == -3 and k.max() == 16
    counts = onp.bincount(k + 3, minlength=20)
    chi2 = float(((counts - n / 20) ** 2 / (n / 20)).sum())
    assert chi2 < 60  # 19 degrees of freedom
    a, b = rb.random.rand(1000).asarray(), rb.random.rand(1000).asarray()
    assert not onp.array_equal(a, b)
    rb.random.seed(123)
    assert onp.array_equal(rb.random.random(n).asarray(), u)


def test_the_reference_testrandom_line(engine):
    import ramba_b200 as rb

    x = rb.random.RandomState(1337).normal(loc=5.0, size=(1000, 10))
    assert x.shape == (1000, 10) and x.dtype == onp.float64
    a = x.asarray()
    assert abs(a.mean() - 5.0) < 0.05
    g = rb.random.default_rng(3)
    assert g.random((4, 5)).shape == (4, 5) and g.normal(size=7).dtype == onp.float64
    assert g.uniform(2.0, 3.0, 9).asarray().min() >= 2.0
    assert g.integers(5, size=11).asarray().max() < 5
    assert isinstance(rb.random.random(), float) and isinstance(rb.random.RandomState(1).randn(), float)


def test_invalid_input(engine):
    import ramba_b200 as rb

    with pytest.raises(ValueError):
        rb.random.uniform(2.0, 1.0, 10)
    with pytest.raises(ValueError):
        rb.random.randint(5, 5, 10)
    with pytest.raises(ValueError):
        rb.random.randint(0, 1 << 63, 10)
    with pytest.raises(ValueError):
        rb.random.seed(-1)
    with pytest.raises(ValueError):
        rb.random.default_rng(-5)
    with pytest.raises(NotImplementedError, match="shuffle"):
        rb.random.RandomState(1).shuffle


# ---------------------------------------------------------------------------------------------------------------------
# plan selection (rb200_describe_plan: no device needed)
def _plan(plans):
    return dict(kv.split("=", 1) for kv in plans[-1].split() if "=" in kv)


def test_plain_draws_plan_on_the_fill_kernel(engine):
    import ramba_b200 as rb

    plans = engine
    cases = [
        (lambda s: rb.random.random(s), "uniform64", "0"),
        (lambda s: rb.random.random(s, dtype=onp.float32), "uniform32", "0"),
        (lambda s: rb.random.standard_normal(s), "normal64", "0"),
        (lambda s: rb.random.normal(1.0, 2.0, s), "normal64", "2"),
        (lambda s: rb.random.uniform(1.0, 2.0, s), "uniform64", "2"),
        (lambda s: rb.random.randint(0, 9, s), "integer", "0"),
        (lambda s: rb.random.randint(-4, 9, s), "integer", "1"),
    ]
    for shape in [(10007,), (101, 33), (9, 8, 7)]:
        for make, form, tail in cases:
            a = make(shape)
            a.asarray()
            d = _plan(plans)
            assert d["kernel"] == "rng_fill" and d["form"] == form and d["tail"] == tail, plans[-1]
            assert d["ndim"] == str(len(shape)) and int(d["inner"]) == shape[-1]


def test_fused_draws_plan_on_the_interpreter(engine):
    import ramba_b200 as rb

    plans = engine
    (rb.random.rand(5000) * rb.arange(5000)).asarray()
    assert _plan(plans)["kernel"] == "general_interpreter"
    float((rb.random.rand(5000) < 0.5).astype(onp.int64).sum())
    assert _plan(plans)["kernel"] == "general_interpreter"
    a = rb.zeros((50, 40))
    a[::2, :] = rb.random.rand(25, 40)
    a.asarray()
    assert any("kernel=general_interpreter" in p for p in plans[-3:])


def test_rng_kill_switch_falls_back_to_the_interpreter():
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import _oracle_backend\n"
            "import ramba_b200 as rb\n"
            "_oracle_backend.install()\n"
            "rb.random.seed(1); rb.random.random((30, 20)).asarray()\n"
            "print(_oracle_backend.PLANS[-1])\n") % (ROOT, HERE)
    env = dict(os.environ, RB200_NO_RNG="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, check=True).stdout
    assert "kernel=general_interpreter" in out, out


def _philox_op(form=0, ctype=0):
    """views[0][0:10] = PHILOX(IOTA 0, key) in float64 (the uniform64 form)."""
    from ramba_b200 import _cabi

    f = _cabi.FusedOp()
    f.abi_version = _cabi.ABI_VERSION
    f.ndim, f.n_views, f.n_insns, f.n_scalars, f.num_workers = 1, 1, 1, 2, 1
    f.itershape[0] = 10
    f.views[0].base = 0x1000  # never dereferenced
    f.views[0].stride[0] = 1
    f.views[0].dtype = _cabi.F64
    f.scalars[0] = 12345
    f.scalars[1] = 10
    i = f.insns[0]
    i.op, i.ctype, i.a_kind, i.a_idx, i.b_kind, i.b_idx, i.imm = _cabi.OP["PHILOX"], ctype, _cabi.K_IOTA, 0, _cabi.K_SCAL, 0, form
    i.st_reg = i.st2 = i.mask_reg = _cabi.NOSTORE
    i.st_view = 0
    return f


def test_malformed_philox_is_rejected_by_run_and_describe():
    import ctypes as C

    from ramba_b200 import _cabi

    lib = _cabi.load()

    def integer(f):
        f.insns[0].imm, f.insns[0].ctype = _cabi.PHILOX_INTEGER, _cabi.T_I64

    def bound(v):
        def m(f):
            integer(f)
            f.insns[0].c_kind, f.insns[0].c_idx = _cabi.K_SCAL, 1
            f.scalars[1] = v & 0xFFFFFFFFFFFFFFFF
        return m

    cases = [
        (lambda f: setattr(f.insns[0], "imm", 4), "philox: bad output form"),
        (lambda f: setattr(f.insns[0], "ctype", _cabi.T_F32), "philox: compute class does not match the output form"),
        (lambda f: setattr(f.insns[0], "b_kind", _cabi.K_IOTA), "philox: the key must be a scalar"),
        (lambda f: setattr(f.insns[0], "a_kind", _cabi.K_SCAL), "philox: the index must be"),
        (integer, "philox: the integer form needs a scalar bound"),
        (bound(0), "philox: the bound must be positive"),
        (bound(-3), "philox: the bound must be positive"),
    ]
    buf = C.create_string_buffer(600)
    for mutate, reason in cases:
        f = _philox_op()
        mutate(f)
        rc_run = lib.rb200_run_deferred_ops(C.byref(f), None)
        msg_run = lib.rb200_last_error().decode()
        rc_desc = lib.rb200_describe_plan(C.byref(f), buf, 600)
        msg_desc = lib.rb200_last_error().decode()
        assert rc_run != 0 and rc_desc != 0 and reason in msg_run and msg_run == msg_desc, (reason, msg_run, msg_desc)
    f = _philox_op()
    assert _cabi.describe_plan(f).startswith("kernel=rng_fill form=uniform64")
    bound(7)(f)
    f.views[0].dtype = _cabi.I64
    assert _cabi.describe_plan(f).startswith("kernel=rng_fill form=integer")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: CUDA against the contract
NORMAL_ATOL = 1e-13


def _gpu_run(tmp_path, name, no_rng):
    env = dict(os.environ)
    env.pop("RB200_NO_RNG", None)
    if no_rng:
        env["RB200_NO_RNG"] = "1"
    out = str(tmp_path / name)
    p = subprocess.run([sys.executable, os.path.join(HERE, "_random_worker.py"), out, "gpu"], env=env, capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    return dict(onp.load(out))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_cuda_draws_match_the_contract(tmp_path):
    from ramba_b200 import random as R

    import _random_worker as W

    fill = _gpu_run(tmp_path, "fill.npz", False)
    interp = _gpu_run(tmp_path, "interp.npz", True)
    assert set(fill) == set(interp)
    for k in fill:  # fill kernel and interpreter: the same bits, normals included; both runs alike
        assert fill[k].dtype == interp[k].dtype and onp.array_equal(fill[k], interp[k]), k
        assert onp.array_equal(fill[k], fill[k[:-1] + ("1" if k.endswith("0") else "0")]), k
    worst = 0.0
    for si, shape in enumerate(W.GPU_SHAPES):
        lin = onp.arange(int(onp.prod(shape))).reshape(shape)
        seed = 100 + si
        g = lambda k: fill["gpu_forms.%s_%d.0" % (k, si)]  # noqa: E731
        assert onp.array_equal(g("u64"), P.draw(lin, R.draw_key(seed, 0), P.UNIFORM64))
        assert onp.array_equal(g("u32"), P.draw(lin, R.draw_key(seed, 1), P.UNIFORM32))
        z = P.draw(lin, R.draw_key(seed, 2), P.NORMAL64)
        err = float(onp.max(onp.abs(g("n64") - z)))
        worst = max(worst, err)
        assert err <= NORMAL_ATOL, (shape, err)
        assert onp.array_equal(g("int"), -7 + P.draw(lin, R.draw_key(seed, 3), P.INTEGER, 1007))
        aff = 3.0 + 0.5 * P.draw(lin, R.draw_key(seed, 4), P.NORMAL64)
        assert float(onp.max(onp.abs(g("aff") - aff))) <= NORMAL_ATOL
    print("largest |normal - oracle| = %.3g" % worst)


@pytest.mark.gpu
def test_cuda_fused_monte_carlo(gpu_engine):
    import ramba_b200 as rb
    from ramba_b200 import random as R

    n = 3_000_001
    rb.random.seed(77)
    inside = int(((rb.random.rand(n) ** 2 + rb.random.rand(n) ** 2) < 1.0).astype(onp.int64).sum())
    x = P.draw(onp.arange(n), R.draw_key(77, 0), P.UNIFORM64)
    y = P.draw(onp.arange(n), R.draw_key(77, 1), P.UNIFORM64)
    assert inside == int(((x ** 2 + y ** 2) < 1.0).sum())
