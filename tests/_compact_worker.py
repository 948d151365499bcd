"""nonzero / flatnonzero / extract programs, run as one rank of a world: `_compact_worker.py OUT` with RANK / WORLD_SIZE in
the environment runs them through the NumPy restatement of the kernels (_compact_vm) over gloo, `_compact_worker.py OUT
cuda` through the CUDA library over NCCL (one GPU per rank, LOCAL_RANK); rank 0 saves the results and the transfer
counters to OUT."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402


def programs():
    """(name, condition builder, values builder or None): the default partitions, partitions that cut the last axis (many
    short runs per rank), views, a broadcast condition, a lazy condition, and densities 0, sparse, 1/2 and all."""
    r = onp.random.default_rng(5)
    x = r.standard_normal((40, 37))
    x[r.random(x.shape) < 0.1] = -0.0
    x[r.random(x.shape) < 0.05] = onp.nan
    sparse = onp.where(r.random((64, 48)) < 0.02, r.integers(1, 9, (64, 48)), 0).astype(onp.int32)
    yield "half", lambda rb: rb.fromarray(x) > 0, lambda rb: rb.fromarray(x)
    yield "float", lambda rb: rb.fromarray(x), lambda rb: rb.fromarray(x * 3)
    yield "sparse", lambda rb: rb.fromarray(sparse), lambda rb: rb.fromarray(sparse)
    yield "none", lambda rb: rb.fromarray(onp.zeros((30, 20))), None
    yield "all", lambda rb: rb.fromarray(onp.ones(1000, dtype=onp.int16)), None
    yield "cols", lambda rb: rb.fromarray(onp.ascontiguousarray(x.T)).T, lambda rb: rb.fromarray(onp.ascontiguousarray(x.T)).T
    yield "lastcut", lambda rb: rb.fromarray(onp.ascontiguousarray(sparse[:3])), None
    yield "step", lambda rb: rb.fromarray(x)[::2, 1::3], lambda rb: rb.fromarray(x * 2)[::2, 1::3]
    yield "bcast", lambda rb: rb.broadcast_to(rb.fromarray(sparse[:1]), (16, 48)), None
    yield "cube", lambda rb: rb.fromarray(sparse.reshape(8, 8, 48)), lambda rb: rb.fromarray(sparse.reshape(8, 8, 48) * 2)


def main():
    import faulthandler

    import _compact_vm
    import _oracle_backend

    faulthandler.dump_traceback_later(int(os.environ.get("RB200_MR_WATCHDOG", "240")), exit=True)
    if (sys.argv[2] if len(sys.argv) > 2 else "oracle") == "oracle":
        _compact_vm.extend_oracle_backend()
        _oracle_backend.install()
    import ramba_b200 as rb
    from ramba_b200 import common
    from ramba_b200.runtime import RT

    if common.num_workers > 1:
        RT.ensure_process_group()
    groups = [0]  # grouped send / receive calls that moved something
    p2p = RT.p2p

    def counted(ops):
        groups[0] += bool(ops)
        return p2p(ops)

    RT.p2p = counted
    res = {}
    for name, cond, vals in programs():
        C = cond(rb)
        V = vals(rb) if vals else None
        rb.sync()
        calls = [("nonzero", lambda: rb.nonzero(C)), ("flatnonzero", lambda: (rb.flatnonzero(C),))]
        if V is not None:
            calls.append(("extract", lambda: (rb.extract(C, V),)))
        for f, call in calls:
            c0, b0, p0 = RT.collectives, RT.bytes_sent, groups[0]
            outs = call()
            c1, p1 = RT.collectives, groups[0]
            for i, o in enumerate(outs):
                res["%s.%s.%d" % (name, f, i)] = o.asarray()
            res["%s.%s.counters" % (name, f)] = onp.array([c1 - c0, p1 - p0, RT.bytes_sent - b0])
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
