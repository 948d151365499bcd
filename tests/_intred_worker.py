"""Integer and truth reductions run as one rank of a world: `_intred_worker.py OUT` with RANK / WORLD_SIZE in the
environment runs them through the oracle backend over gloo.  Rank 0 saves every result and the blocks each rank held of
every source array to OUT.  The data come from test_integer_reductions' generators, so every rank holds the same values;
the rank-boundary cases place their extreme, nonzero or zero at the first and last element of every rank's block."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402

import test_integer_reductions as T  # noqa: E402


def _blocks(A):
    """[[start..., size...] per rank] of A's distribution (global coordinates)."""
    return onp.array([[int(s) for s in sv.start] + [int(s) for s in sv.size] for sv in A.distribution], dtype=onp.int64)


def _run(rb, A, op, axis):
    if op == "cumsum":
        return rb.cumsum(A, axis=axis)
    if op == "mean":
        return A.mean(axis=axis)
    return getattr(rb, op)(A, axis=axis)


def main():
    import faulthandler

    import _oracle_backend

    faulthandler.dump_traceback_later(int(os.environ.get("RB200_MR_WATCHDOG", "240")), exit=True)
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
            r = _run(rb, A, op, axis)
            res["%s.%s.%s" % (name, op, axis)] = onp.asarray(r.asarray() if isinstance(r, rb.ndarray) else r)
    n = 4001
    edges = set()
    for b in _blocks(rb.fromarray(onp.zeros(n, dtype=onp.int64))):
        if b[1] > 0:
            edges |= {int(b[0]), int(b[0] + b[1] - 1)}
    for p in sorted(edges):
        for what, dts in (("min", (onp.int64, onp.uint32, onp.int8, onp.uint8)), ("max", (onp.int64, onp.uint32, onp.int16, onp.uint16)),
                          ("any", (onp.int64, onp.uint8, onp.bool_)), ("all", (onp.int32, onp.uint8, onp.bool_))):
            for dt in dts:
                r = getattr(rb.fromarray(T.edge_data(what, dt, n, p)), what)()
                res["edge.%s.%s.%d" % (what, onp.dtype(dt).name, p)] = onp.asarray(r)
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
