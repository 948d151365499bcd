"""Worker process of the multi-rank CPU tests: RANK/WORLD_SIZE come from the environment (the same
variables torchrun sets); collectives run over gloo, op lists through the oracle."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402

MODE = sys.argv[2] if len(sys.argv) > 2 else "oracle"
if MODE == "oracle":
    import _oracle_backend  # noqa: E402

    _oracle_backend.install()

import _programs  # noqa: E402
import ramba_b200 as rb  # noqa: E402
from ramba_b200 import common  # noqa: E402
from ramba_b200.runtime import RT  # noqa: E402


def main():
    names = sys.argv[1].split(",")
    # a rank that dies or deadlocks leaves the others waiting in a collective: every rank dumps its Python stack and exits
    # after WATCHDOG seconds, so that a hang shows up as a failed test with the place it hung at, not as a timeout
    import faulthandler

    faulthandler.dump_traceback_later(int(os.environ.get("RB200_MR_WATCHDOG", "240")), exit=True)
    RT.ensure_process_group()
    failures = []
    import test_api_parity
    import test_edges

    import _random_programs

    import test_scan_kernel
    import test_stencil_tile
    import test_stream_kernel

    import _dag_fuzz
    import _expr_fuzz
    import _limit_fuzz
    import test_reshape_copy

    progs = (list(_programs.ALL) + list(test_api_parity.CASES) + [test_edges._ragged, test_edges._empty, test_edges._dtypes]
             + (_random_programs.CASES if os.environ.get("RB200_MR_ALL_RANDOM") else _random_programs.CASES[:12])
             + (_dag_fuzz.CASES[:60] if os.environ.get("RB200_MR_ALL_RANDOM") else _dag_fuzz.CASES[:10])
             + (_limit_fuzz.CASES[:40] if os.environ.get("RB200_MR_ALL_RANDOM") else _limit_fuzz.CASES[:6])
             + (_expr_fuzz.CASES[:60] if os.environ.get("RB200_MR_ALL_RANDOM") else _expr_fuzz.CASES[:8])
             + (_expr_fuzz.TRIG_CASES[:40] if os.environ.get("RB200_MR_ALL_RANDOM") else _expr_fuzz.TRIG_CASES[:6])
             + (_expr_fuzz.VIEW_CASES[:60] if os.environ.get("RB200_MR_ALL_RANDOM") else _expr_fuzz.VIEW_CASES[:8])
             + (_expr_fuzz.API_CASES[:60] if os.environ.get("RB200_MR_ALL_RANDOM") else _expr_fuzz.API_CASES[:6])
             + (_expr_fuzz.SHAPE_CASES[:60] if os.environ.get("RB200_MR_ALL_RANDOM") else _expr_fuzz.SHAPE_CASES[:8])
             + (_expr_fuzz.SKELETON_CASES[:50] if os.environ.get("RB200_MR_ALL_RANDOM") else _expr_fuzz.SKELETON_CASES[:6])
             + (_expr_fuzz.PARTITION_CASES[:60] if os.environ.get("RB200_MR_ALL_RANDOM") else _expr_fuzz.PARTITION_CASES[:10])
             + (_expr_fuzz.REDUCTION_CASES[:50] if os.environ.get("RB200_MR_ALL_RANDOM") else _expr_fuzz.REDUCTION_CASES[:8])
             + (_expr_fuzz.MIXED_CASES[:60] if os.environ.get("RB200_MR_ALL_RANDOM") else _expr_fuzz.MIXED_CASES[:10])
             + [test_reshape_copy.reshape_programs])
    # the stencil programs restate the engine's per-operation classes on the NumPy side: bit for bit across ranks.  The
    # streaming / scan kernel programs: float32 arrays with Python-float weights are computed in float64 by the op list
    # (Numba's typing) but in float32 by NumPy, so these compare with a dtype tolerance
    exact, loose = [], []
    for (nm, fn) in list(test_stencil_tile.CASES) + list(test_stream_kernel.CASES):
        def f(np, fn=fn):
            return fn(np)
        f.__name__ = nm
        (exact if (nm, fn) in test_stencil_tile.CASES else loose).append(f)

    def scan_small(np):
        return test_scan_kernel.scans(np, False)

    if os.environ.get("RB200_MR_NPY"):
        def load_npy(np):
            # every rank reads only its own block of the file (ramba_b200.load); NumPy reads it whole
            x = np.load(os.environ["RB200_MR_NPY"])
            return [onp.asarray(x.asarray() if hasattr(x, "asarray") else x), onp.asarray(float((x * 2.0).sum()))]

        progs.append(load_npy)

    loose.append(scan_small)
    for prog in progs + exact + loose:
        if prog.__name__ not in names and names != ["all"]:
            continue
        if os.environ.get("RB200_MR_TRACE"):
            print("RANK %d: %s" % (common.worker_num, prog.__name__), flush=True)
        try:
            got = prog(rb)
        except BaseException:
            import traceback

            print("RANK %d failed in %s:\n%s" % (common.worker_num, prog.__name__, traceback.format_exc()), flush=True)
            os._exit(3)  # (the other ranks are released by their watchdogs)
        exp = prog(onp)
        # a second run of the same program meets the memoised flush scripts (pack -> transfers -> ranges replayed from the
        # tape of the first run): it must give the same values
        again = prog(rb)
        if len(again) != len(got) or not all(onp.array_equal(onp.asarray(a), onp.asarray(b), equal_nan=True)
                                              if onp.asarray(a).dtype.kind in "fc" else onp.array_equal(onp.asarray(a), onp.asarray(b))
                                              for a, b in zip(again, got)):
            failures.append("%s (second run differs from the first)" % prog.__name__)
        for i, (g, e) in enumerate(zip(got, exp)):
            g, e = onp.asarray(g), onp.asarray(e)
            if prog in exact:
                ok = g.shape == e.shape and g.dtype == e.dtype and onp.array_equal(onp.ascontiguousarray(g).view(onp.uint8), onp.ascontiguousarray(e).view(onp.uint8))
            elif prog in loose:
                tol = 1e-5 if e.dtype == onp.float32 else 1e-12
                ok = g.shape == e.shape and g.dtype == e.dtype and (onp.allclose(g, e, rtol=tol, atol=tol) if e.dtype.kind == "f" else onp.array_equal(g, e))
            else:
                ok = g.shape == e.shape and (onp.allclose(g, e, rtol=1e-13, atol=1e-12 if prog.__name__.startswith(("random_program", "dag_program", "limit_program", "expr_program", "trig_mask_program", "view_program", "api_program", "shape_program", "skeleton_program", "partition_program", "reduction_program", "mixed_program")) else 1e-15) if e.dtype.kind == "f" else onp.array_equal(g, e))
            if not ok:
                failures.append("%s[%d]" % (prog.__name__, i))
    if MODE == "cuda":
        from ramba_b200 import _cabi

        assert RT.is_cuda and _cabi.launch_count() > 0, "the CUDA library did not run"
    if MODE == "oracle" and os.environ.get("RB200_DUMP_PLANS"):
        # debugging aid: which kernel of the CUDA library every op list of this rank would have got
        with open("%s.%d" % (os.environ["RB200_DUMP_PLANS"], common.worker_num), "w") as f:
            f.write("\n".join(_oracle_backend.PLANS) + "\n")
    print("RANK %d/%d launches=%d bytes_sent=%d collectives=%d ring_receives=%d failures=%s" % (common.worker_num, common.num_workers, RT.launches, RT.bytes_sent, RT.collectives, RT.ring_receives, failures))
    sys.stdout.flush()
    import torch.distributed as dist

    dist.barrier()
    faulthandler.cancel_dump_traceback_later()
    dist.destroy_process_group()
    sys.exit(1 if failures else 0)


if __name__ == "__main__":
    main()
