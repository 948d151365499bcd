"""Accumulation programs run as one rank of a world: `_accum_worker.py OUT` with RANK / WORLD_SIZE in the environment runs
them through the oracle backend over gloo, `_accum_worker.py OUT cuda` through the CUDA library over NCCL (one GPU per
rank, LOCAL_RANK).  Rank 0 saves every result, the blocks each rank held of every source array, and the collectives
each float32 sum took, to OUT.  The data are built from test_reduction_accuracy's generators, so every rank holds the
same values."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402

import test_reduction_accuracy as T  # noqa: E402


def _blocks(A):
    """[[start..., size...] per rank] of A's distribution (global coordinates)."""
    return onp.array([[int(s) for s in sv.start] + [int(s) for s in sv.size] for sv in A.distribution], dtype=onp.int64)


def main():
    import faulthandler

    import _oracle_backend

    faulthandler.dump_traceback_later(int(os.environ.get("RB200_MR_WATCHDOG", "240")), exit=True)
    if (sys.argv[2] if len(sys.argv) > 2 else "oracle") == "oracle":
        _oracle_backend.install()
    import ramba_b200 as rb
    from ramba_b200 import common
    from ramba_b200.runtime import RT

    if common.num_workers > 1:
        RT.ensure_process_group()
    res = {}
    for name, x, ops in T.world_sources():
        A = rb.fromarray(x)
        rb.sync()
        res[name + ".blocks"] = _blocks(A)
        for op, axis in ops:
            key = "%s.%s.%s" % (name, op, axis)
            c0 = RT.collectives
            if op in ("scummin", "scummax"):
                f = onp.minimum if op == "scummin" else onp.maximum
                r = rb.scumulative(f, f, A, axis=axis)
            elif op == "cumsum":
                r = rb.cumsum(A, axis=axis)
            else:
                r = getattr(rb, op)(A, axis=axis)
            out = onp.asarray(r.asarray() if isinstance(r, rb.ndarray) else r)
            res[key] = out
            res[key + ".collectives"] = onp.array([RT.collectives - c0])
    rb.sync()
    if common.worker_num == 0:
        onp.savez(sys.argv[1], **res)
    if common.num_workers > 1:
        import torch.distributed as dist

        dist.barrier()
        dist.destroy_process_group()
    print("ok rank=%d" % common.worker_num)


if __name__ == "__main__":
    main()
