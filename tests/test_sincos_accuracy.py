"""float64 sin / cos of the general interpreter, in ulps against 200-bit references.

Every float64 SIN, COS and SINCOS of the interpreter kernels runs sincos_v (rb200_vm.cuh): a Cody-Waite reduction and
fdlibm polynomials for the V elements a thread holds, unless one of those V is NaN, Inf or at least 1e9 in magnitude:
then all V take the CUDA library's sincos.  These tests run both paths on every kernel that calls it - the lean 1-D
kernel, the full 1-D kernel (RB200_NO_LEAN_INTERP=1, read once per process: a subprocess), the N-d kernel (V = 4) and the
generic decode path - each checked through rb200_describe_plan to be the kernel it is named for, and hold each path to its
own bound: BOUND_OURS for sincos_v, 2 ulp (CUDA's documented bound for double sin / cos) for the library.  Zeros of
either sign, tiny arguments (sin(x) is x, cos(x) is 1), Inf and NaN are compared bit for bit.  float32 arrays: in
float64 arithmetic (a Python-float operand, the result rounded to float32 on store) within half an ulp plus 2^-28
relative, in the float32 class (the library's sincosf) within 2 ulp."""
import functools
import json
import os
import subprocess
import sys

import mpmath
import numpy as onp
import pytest
from mpmath import libmp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")

PREC = 200          # bits of the references
BOUND_OURS = 1.55   # ulp, sincos_v; the largest error over these sets, on an H100: 1.5126 (sin), 1.5130 (cos)
BOUND_LIB = 2.0     # ulp, the CUDA library's sin / cos
BOUND_F32 = 2.0     # ulp of float32, the CUDA library's sincosf
TINY = 2.0 ** -27   # below this sin(x) rounds to x and cos(x) to 1
SWITCH = 1.0e9      # |x| from which sincos_v hands its V elements to the library

LANES = 256         # threads per CTA: element e of a tile is held by thread e % 256, with e + 256, e + 512, ...
TILE = LANES * 8    # the 1-D kernels' tile (V = 8); the N-d kernel's tile (V = 4) divides it


# ---- arguments --------------------------------------------------------------------------------------------------------
def _both_signs(x):
    x = onp.asarray(x, dtype=onp.float64)
    return onp.concatenate([x, -x])


def _alternate_signs(x):
    x = onp.array(x, dtype=onp.float64)
    x[1::2] *= -1.0
    return x


def _steps(x, n):
    """x and its n neighbours on either side, in ulps"""
    up, down = [x], [x]
    for _ in range(n):
        up.append(onp.nextafter(up[-1], onp.inf))
        down.append(onp.nextafter(down[-1], -onp.inf))
    return onp.array(down[:0:-1] + up)


HARD = [  # sin, then cos: 1.50 - 1.513 ulp
    "0x1.9b7655c28f5c3p+16", "-0x1.faef0972954c1p+27", "0x1.8b96df5c28f5cp+17", "0x1.4ae769999999ap+17", "0x1.4f2b8e3d70a3ep+19",
    "0x1.23ac8eb851eb8p+18", "0x1.c54e7d70a3d71p+19", "-0x1.23beb7300c12cp+17",
    "0x1.19efac28f5c29p+17", "0x1.d18c6cccccccdp+19", "0x1.e0d1be8f5c290p+19", "0x1.7324f028f5c29p+19", "0x1.5a9f21eb851ecp+17",
    "0x1.fb249c28f5c29p+17", "0x1.8183be3d70a3ep+19",
]


@functools.lru_cache(None)
def argument_sets():
    """name -> float64 arguments, seeded; "ours" sets are finite with |x| < 1e9, "library" sets are not"""
    rng = onp.random.default_rng(20261017)
    n = 8000
    ours = {
        "uniform [0, pi/4]": _alternate_signs(rng.uniform(0.0, onp.pi / 4, n)),
        "uniform [0, 10]": _alternate_signs(rng.uniform(0.0, 10.0, n)),
        "uniform [0, 1e6]": _alternate_signs(rng.uniform(0.0, 1e6, n)),
        "uniform [1e6, 1e9)": _alternate_signs(rng.uniform(1e6, 1e9, n)),
    }
    # the headline chain's arguments, arange(N) * 0.001: blocks spread over the first 1e9 elements
    starts = onp.unique(onp.concatenate([[0], onp.geomspace(1e3, 1e9 - 256, 31).astype(onp.int64)]))
    ours["config 2 blocks"] = _alternate_signs(onp.concatenate([onp.arange(s, s + 256, dtype=onp.int64) for s in starts]) * 0.001)
    # the nearest doubles to k * pi / 2, where the reduction cancels most, and their neighbours
    ks = onp.unique(onp.concatenate([onp.arange(1, 3001), onp.geomspace(3001, 6e8, 3000).astype(onp.int64)]))
    with mpmath.workprec(PREC):
        near = onp.array([float(mpmath.mpf(int(k)) * mpmath.pi / 2) for k in ks])
    ours["k pi/2"] = _both_signs(onp.concatenate([near, onp.nextafter(near, onp.inf), onp.nextafter(near, -onp.inf)]))
    # where sincos_v errs most among 3e8 arguments swept (every 5th of arange(1e9) * 0.001; uniform below 1e9)
    ours["largest errors found"] = _both_signs([float.fromhex(h) for h in HARD])
    at = _steps(SWITCH, 4)
    ours["below 1e9"] = _both_signs(at[at < SWITCH])
    ours["tiny"] = _both_signs(onp.concatenate([[0.0, 5e-324, 1e-300, 2.0 ** -30], 2.0 ** onp.linspace(-1074, -28, 48), [onp.nextafter(TINY, 0.0)]]))
    library = {
        "from 1e9": _both_signs(at[at >= SWITCH]),
        "large": _both_signs([1e10, 1e15, 1e22, 2.0 ** 1000, onp.finfo(onp.float64).max]),
        "inf and nan": onp.array([onp.inf, -onp.inf, onp.nan]),
    }
    return ours, library


@functools.lru_cache(None)
def arguments():
    """(all arguments, how many lead with |x| < 1e9), the order every reference and result table here uses"""
    ours, library = argument_sets()
    x_ours = onp.concatenate(list(ours.values()))
    return onp.concatenate([x_ours] + list(library.values())), x_ours.size


# ---- references and the ulp measure -----------------------------------------------------------------------------------
def _double_double(v):
    hi = libmp.to_float(v, rnd=libmp.round_nearest)
    return hi, libmp.to_float(libmp.mpf_sub(v, libmp.from_float(hi), PREC), rnd=libmp.round_nearest)


def _reference(x):
    """sin and cos of every x at PREC bits as double-doubles: [sin hi, sin lo, cos hi, cos lo] (hi: the exact value
    rounded to float64); NaN where x is not finite"""
    out = onp.full((4, x.size), onp.nan)
    for i, xi in enumerate(x.tolist()):
        if xi - xi == 0.0:
            c, s = libmp.mpf_cos_sin(libmp.from_float(xi), PREC)
            out[0, i], out[1, i] = _double_double(s)
            out[2, i], out[3, i] = _double_double(c)
    return out


@functools.lru_cache(None)
def references():
    """(float64 references of arguments(), references of the same arguments rounded to float32), computed once"""
    x, _ = arguments()
    with onp.errstate(over="ignore"):
        x32 = x.astype(onp.float32).astype(onp.float64)
    return _reference(x), _reference(x32)


def ulp_error(got, hi, lo, dtype=onp.float64):
    """|got - exact| in ulps of the exact result (hi + lo) rounded to dtype; the ulp of a zero result is dtype's
    smallest subnormal.  NaN where got is NaN."""
    got = onp.asarray(got, dtype=onp.float64)
    ulp = onp.spacing(onp.abs(hi.astype(dtype))).astype(onp.float64)
    with onp.errstate(invalid="ignore"):
        return onp.abs((got - hi) - lo) / ulp


# ---- placements -------------------------------------------------------------------------------------------------------
PROGRAMS = {
    # name: (outputs from (X, X32), what each output is)
    "sin": (lambda rb, X, X32: [rb.sin(X)], ["sin"]),
    "cos": (lambda rb, X, X32: [rb.cos(X)], ["cos"]),
    # sin and cos of one operand: SINCOS; imm 0 keeps sin and parks cos, imm 1 the other way round; the parked half is
    # stored straight to its view, or (times 1.0) read back from its register
    "sincos": (lambda rb, X, X32: [rb.sin(X), rb.cos(X)], ["sin", "cos"]),
    "cossin": (lambda rb, X, X32: [rb.cos(X), rb.sin(X)], ["cos", "sin"]),
    "sincos read back": (lambda rb, X, X32: [rb.sin(X), rb.cos(X) * 1.0], ["sin", "cos"]),
    # float32 class: the library's sincosf
    "sin f32": (lambda rb, X, X32: [rb.sin(X32)], ["sin f32"]),
    "cos f32": (lambda rb, X, X32: [rb.cos(X32)], ["cos f32"]),
    "sincos f32": (lambda rb, X, X32: [rb.sin(X32), rb.cos(X32)], ["sin f32", "cos f32"]),
    # float32 arrays in float64 arithmetic, rounded to float32 on store
    "f32 in f64": (lambda rb, X, X32: [rb.sin(X32 * 1.0), rb.cos(X32 * 1.0)], ["sin f32 in f64", "cos f32 in f64"]),
}
SINCOS_FORM = {"sincos": (0, True), "cossin": (1, True), "sincos read back": (0, False), "sincos f32": (0, True)}  # imm, parked half stored
PLACEMENTS = {
    "lean": ["sin", "cos", "sincos", "cossin", "sincos read back", "sin f32", "sincos f32"],
    "full": list(PROGRAMS),
    "nd": list(PROGRAMS),
    # the trigonometric instruction itself must read a view without a prefetch slot: SINCOS reads the accumulator
    "generic": ["sin", "cos", "sin f32", "cos f32"],
}
TRIG = ("SIN", "COS", "SINCOS")


def _place(placement, x):
    """x (a multiple of TILE elements) as the operand of `placement`: float64 and float32 arrays, and for the generic
    path two more float64 arrays that take the prefetch slots of the 1-D kernel first"""
    import ramba_b200 as rb

    with onp.errstate(over="ignore"):
        x32 = x.astype(onp.float32)
    if placement == "nd":  # rows of TILE elements in a wider array: a 2-D view that does not collapse to 1-D
        w, w32 = onp.zeros((x.size // TILE, TILE + 8)), onp.zeros((x.size // TILE, TILE + 8), dtype=onp.float32)
        w[:, :TILE], w32[:, :TILE] = x.reshape(-1, TILE), x32.reshape(-1, TILE)
        return rb.fromarray(w)[:, :TILE], rb.fromarray(w32)[:, :TILE], []
    slot_takers = [rb.zeros(x.size), rb.zeros(x.size)] if placement == "generic" else []
    return rb.fromarray(x), rb.fromarray(x32), slot_takers


def _evaluate(placement, arrays):
    """Every program of `placement` on every array: ({"program|array|i": output i as a flat NumPy array},
    [[program, plan, [[opcode, imm, parked half stored], ...]], ...] of the op lists they ran)"""
    import ramba_b200 as rb
    from ramba_b200 import _cabi
    from ramba_b200.runtime import RT

    results, plans = {}, []
    for aname, x in arrays.items():
        X, X32, slot_takers = _place(placement, x)
        rb.sync()
        for prog in PLACEMENTS[placement]:
            make, _ = PROGRAMS[prog]
            be = RT.be()
            run = be.run

            def record(fop, stream=None, prog=prog):
                insns = [[_cabi.OPS[fop.insns[i].op], int(fop.insns[i].imm), fop.insns[i].c_kind == _cabi.K_VIEW] for i in range(fop.n_insns)]
                plans.append([prog, _cabi.describe_plan(fop), insns])
                return run(fop, stream)

            be.run = record
            try:
                keep = slot_takers[0] + slot_takers[1] if slot_takers else None  # reads both before the trigonometric operand
                outs = make(rb, X, X32)
                rb.sync()
            finally:
                be.run = run
            for i, o in enumerate(outs):
                results["%s|%s|%d" % (prog, aname, i)] = o.asarray().reshape(-1)
            del keep, outs
    return results, plans


def _generic_pcs(plan):
    for f in plan.split():
        if f.startswith("generic="):
            return {int(i) for i in f[len("generic="):].split(",")}
    return set()


def check_plans(placement, plans):
    """every op list of `placement` that computes sin / cos ran on the kernel and path the placement is named for"""
    seen = set()
    for prog, plan, insns in plans:
        trig = [pc for pc, ins in enumerate(insns) if ins[0] in TRIG]
        if not trig:
            continue
        seen.add(prog)
        where = (placement, prog, plan, insns)
        assert plan.startswith("kernel=general_interpreter form=elementwise "), where
        generic = _generic_pcs(plan)
        if placement == "lean":
            assert plan.endswith(" variant=lean"), where
        elif placement == "full":
            assert " ndim=1 " in plan and "variant=lean" not in plan and not generic & set(trig), where
        elif placement == "nd":
            assert " ndim=2 " in plan and not generic & set(trig), where
        else:
            assert " ndim=1 " in plan and set(trig) <= generic, where
        if prog in SINCOS_FORM:
            sincos = [insns[pc] for pc in trig if insns[pc][0] == "SINCOS"]
            assert sincos and all((imm, stored) == SINCOS_FORM[prog] for _, imm, stored in sincos), where
    assert seen == set(PLACEMENTS[placement]), (placement, sorted(seen))


# ---- what each element must hold --------------------------------------------------------------------------------------
def _lane0(n_values, poison):
    """a multiple of TILE elements with value slots where every thread of every tile holds its first element (e % TILE
    < 256): the other V - 1 elements of each slot's thread, in the 1-D tile (V = 8) and the N-d tile (V = 4) alike, are
    `poison`.  Two tiles at least.  Returns the array and the element index of each slot."""
    tiles = max(-(-n_values // LANES), 2)
    a = onp.full((tiles, TILE // LANES, LANES), poison)
    slots = (onp.arange(tiles)[:, None] * TILE + onp.arange(LANES)[None, :]).reshape(-1)[:n_values]
    return a.reshape(-1), slots


@functools.lru_cache(None)
def layout(small=False):
    """name -> (array, element index of each checked value, index of that value in arguments()):
    "ours": the arguments below 1e9 alone, so every thread runs sincos_v; "mates 1e10" / "mates nan": every argument in
    a thread whose other elements are 1e10 / NaN, so every element takes the library routine.  small: two tiles each,
    for plan checks."""
    x, n_ours = arguments()
    if small:
        x, n_ours = x[:LANES], LANES
    out = {}
    ours = onp.full(max(-(-n_ours // TILE), 2) * TILE, 0.5)  # (two rows at least: one would collapse to 1-D)
    ours[:n_ours] = x[:n_ours]
    out["ours"] = (ours, onp.arange(n_ours), onp.arange(n_ours))
    for name, poison in (("mates 1e10", 1e10), ("mates nan", onp.nan)):
        a, slots = _lane0(x.size, poison)
        a[slots] = x
        out[name] = (a, slots, onp.arange(x.size))
    return out


def check_results(placement, results):
    """every checked element within its bound, and the exact cases bit for bit; returns the worst error per output
    kind and path ({(output, path): ulps})"""
    x, _ = arguments()
    ref64, ref32 = references()
    with onp.errstate(over="ignore"):
        x32 = x.astype(onp.float32)
    failures, worst = [], {}
    for aname, (_, slots, which) in layout().items():
        for prog in PLACEMENTS[placement]:
            for i, what in enumerate(PROGRAMS[prog][1]):
                got = results["%s|%s|%d" % (prog, aname, i)][slots]
                xs = x[which]
                fn = what.split()[0]
                row = 0 if fn == "sin" else 2
                where = (placement, prog, aname, what)
                if what in ("sin", "cos"):
                    hi, lo = ref64[row][which], ref64[row + 1][which]
                    err = ulp_error(got, hi, lo)
                    path = "sincos_v" if aname == "ours" else "library"
                    bound = BOUND_OURS if aname == "ours" else BOUND_LIB
                    src, bits = xs, onp.uint64
                    got_bits = got.view(onp.uint64)
                else:
                    hi, lo = ref32[row][which], ref32[row + 1][which]
                    err = ulp_error(got, hi, lo, onp.float32)
                    if what.endswith("in f64"):
                        path, bound = "f32 in f64", rounded_bound(hi)
                    else:
                        path, bound = "sincosf", BOUND_F32
                    src, bits = x32[which], onp.uint32
                    got_bits = got.astype(onp.float32).view(onp.uint32)
                finite = onp.isfinite(src)
                e = err[finite]
                if e.size:
                    worst[fn, path] = max(worst.get((fn, path), 0.0), float(onp.where(onp.isnan(e), onp.inf, e).max()))
                bad = finite & ~(err <= bound)
                if bad.any():
                    j = onp.flatnonzero(bad)[:5]
                    failures.append("%s: %d over %s ulp, e.g. x=%r got=%r err=%r" % (where, bad.sum(), onp.max(bound), src[j].tolist(), got[j].tolist(), err[j].tolist()))
                if (~finite & ~onp.isnan(got)).any():
                    failures.append("%s: not NaN for x=%r" % (where, src[~finite & ~onp.isnan(got)].tolist()))
                tiny = onp.abs(src) < TINY
                want = src[tiny].astype(got.dtype).view(bits) if fn == "sin" else onp.ones(tiny.sum(), got.dtype).view(bits)
                if (got_bits[tiny] != want).any():
                    j = onp.flatnonzero(got_bits[tiny] != want)[:5]
                    failures.append("%s: bits of %s(x) for tiny x=%r are %r, want %r" % (where, fn, src[tiny][j].tolist(), [hex(int(b)) for b in got_bits[tiny][j]],
                                                                                    [hex(int(b)) for b in want[j]]))
    assert not failures, "\n".join(failures)
    return worst


def rounded_bound(hi):
    """a float64 result within 2^-28 of the exact one, rounded to float32: half an ulp plus 2^-28 relative, in ulps"""
    return 0.5 + 2.0 ** -28 * onp.abs(hi) / onp.spacing(onp.abs(hi.astype(onp.float32))).astype(onp.float64)


def _report(placement, worst):
    print("worst error, %s: %s" % (placement, ", ".join("%s %s %.4f ulp" % (fn, path, u) for (fn, path), u in sorted(worst.items()))))


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_the_ulp_measure_holds_glibc_to_one_ulp():
    """the harness itself: glibc's sin / cos are within 1 ulp of the references over every finite argument, their
    float32 roundings within half an ulp, and results 2 ulp away read as 2 ulp"""
    x, _ = arguments()
    ref64, ref32 = references()
    fin = onp.isfinite(x)
    for row, f in ((0, onp.sin), (2, onp.cos)):
        err = ulp_error(f(x[fin]), ref64[row][fin], ref64[row + 1][fin])
        assert err.max() <= 1.0, (f.__name__, x[fin][err.argmax()], err.max())
        away = onp.copysign(onp.inf, ref64[row][fin])  # (toward zero, the ulp may halve)
        off = onp.nextafter(onp.nextafter(ref64[row][fin], away), away)
        err2 = ulp_error(off, ref64[row][fin], ref64[row + 1][fin])
        assert err2.min() >= 1.5 and err2.max() <= 4.5, (f.__name__, err2.min(), err2.max())
        with onp.errstate(over="ignore"):
            x32 = x.astype(onp.float32).astype(onp.float64)
        fin32 = onp.isfinite(x32)
        err32 = ulp_error(f(x32[fin32]).astype(onp.float32), ref32[row][fin32], ref32[row + 1][fin32], onp.float32)
        assert onp.all(err32 <= rounded_bound(ref32[row][fin32])), (f.__name__, err32.max())


def test_the_argument_sets():
    ours, library = argument_sets()
    x, n_ours = arguments()
    assert onp.all(onp.abs(x[:n_ours]) < SWITCH) and not onp.any(onp.abs(x[n_ours:]) < SWITCH)
    for name, s in ours.items():
        assert (s < 0).any() and (s > 0).any(), name
    tiny = ours["tiny"]
    assert onp.signbit(tiny[tiny == 0]).tolist() == [False, True]
    lay = layout()
    for name, (a, slots, which) in lay.items():
        assert a.size % TILE == 0 and onp.array_equal(a[slots], x[which], equal_nan=True), name
        if name != "ours":  # every other element of a value's thread is the poison, in tiles of V = 8 and of V = 4
            e = onp.arange(a.size)
            assert onp.all(e[slots] % TILE < LANES)
            mates = ~onp.isin(e, slots) & (e % TILE >= LANES)
            assert not onp.any(onp.abs(a[mates]) < SWITCH)


def test_every_placement_plans_the_kernel_it_is_named_for(oracle_engine):
    for placement in ("lean", "nd", "generic"):
        _, plans = _evaluate(placement, {k: v[0] for k, v in layout(small=True).items()})
        check_plans(placement, plans)


def test_the_full_kernel_placement_plans_off_the_lean_kernel(tmp_path):
    plans = _run_full(tmp_path, "plans")[1]
    check_plans("full", plans)


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _full_worker(out_dir, mode):
    """The full 1-D kernel's programs in a process of their own (RB200_NO_LEAN_INTERP=1): outputs and plans to out_dir.
    mode "plans": on the oracle backend, one tile per array; "gpu": the product backend (under RB200_DRY_GPU_TESTS=1 the
    oracle, as the gpu_engine fixture does)."""
    from ramba_b200.runtime import RT

    RT.reset()
    if mode == "plans":
        import _oracle_backend

        _oracle_backend.install()
    elif os.environ.get("RB200_DRY_GPU_TESTS"):
        import conftest

        conftest._dry_gpu()
    results, plans = _evaluate("full", {k: v[0] for k, v in layout(small=mode == "plans").items()})
    onp.savez(os.path.join(out_dir, "results.npz"), **results)
    with open(os.path.join(out_dir, "plans.json"), "w") as f:
        json.dump(plans, f)


def _run_full(tmp_path, mode):
    code = "import sys; sys.path[:0] = [%r, %r]; import test_sincos_accuracy as t; t._full_worker(%r, %r)" % (ROOT, HERE, str(tmp_path), mode)
    env = dict(os.environ, RB200_NO_LEAN_INTERP="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    with onp.load(os.path.join(str(tmp_path), "results.npz")) as z:
        results = {k: z[k] for k in z.files}
    with open(os.path.join(str(tmp_path), "plans.json")) as f:
        return results, json.load(f)


@pytest.mark.gpu
@pytest.mark.parametrize("placement", ["lean", "nd", "generic"])
def test_sin_cos_accuracy(gpu_engine, placement):
    results, plans = _evaluate(placement, {k: v[0] for k, v in layout().items()})
    check_plans(placement, plans)
    _report(placement, check_results(placement, results))


@pytest.mark.gpu
def test_sin_cos_accuracy_on_the_full_kernel(gpu_engine, tmp_path):
    results, plans = _run_full(tmp_path, "gpu")
    check_plans("full", plans)
    _report("full", check_results("full", results))
