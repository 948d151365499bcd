"""groupby programs, run as one rank of a world: `_group_worker.py OUT` with RANK / WORLD_SIZE in the environment runs them
through the NumPy restatement of the kernel (_group_vm) over gloo, `_group_worker.py OUT cuda` through the CUDA library
over NCCL (one GPU per rank, LOCAL_RANK); rank 0 saves the results and the transfer counters to OUT."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402

AGGS = ("sum", "prod", "min", "max", "count", "mean", "var", "std", "nanmean")
PASSES = {"sum": 1, "prod": 1, "min": 1, "max": 1, "count": 0, "mean": 1, "var": 2, "std": 2, "nanmean": 2}


def programs():
    """(name, source builder, dim, labels, num_groups): exactly representable data, so that every world agrees bit for bit."""
    r = onp.random.default_rng(5)
    rows = (r.integers(-8, 9, size=(64, 30)) * 0.5).astype(onp.float64)
    yield "rows", lambda rb: rb.fromarray(rows), 1, r.integers(0, 5, size=30), 6            # (space, time) grouped on time
    flat = r.integers(-4, 5, size=301).astype(onp.float64)
    yield "flat", lambda rb: rb.fromarray(flat), 0, onp.arange(301) % 7, 7                  # the grouped axis is cut
    cube = r.integers(-3, 4, size=(10, 24, 9)).astype(onp.int64)
    yield "cube", lambda rb: rb.fromarray(cube), 1, r.integers(0, 4, size=24), 4
    cols = r.integers(-6, 7, size=(40, 50)).astype(onp.float32)
    yield "cols", lambda rb: rb.fromarray(cols), 0, r.integers(0, 3, size=40), 3


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
    for rep in range(2):
        for name, build, dim, labels, G in programs():
            A = build(rb)
            rb.sync()
            gb = A.groupby(dim, labels, G)
            cut = bool(common.num_workers > 1 and gb._axis_cut(A))
            for agg in AGGS:
                c0, b0 = RT.collectives, RT.bytes_sent
                nd = getattr(gb, agg)()
                c1, b1 = RT.collectives, RT.bytes_sent
                out = nd.asarray()
                res["%s.%s.%d" % (name, agg, rep)] = out
                res["%s.%s.%d.counters" % (name, agg, rep)] = onp.array([c1 - c0, b1 - b0, int(cut), out.size, int(A.dtype.kind == "f")])
            res["%s.anomaly.%d" % (name, rep)] = (gb - gb.mean()).asarray()
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
