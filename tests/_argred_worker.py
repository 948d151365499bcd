"""argmax / argmin programs, run as one rank of a world: `_argred_worker.py OUT` with RANK / WORLD_SIZE in the environment
runs them through the NumPy restatement of the kernel (_argred_vm) over gloo, `_argred_worker.py OUT cuda` through the
CUDA library over NCCL (one GPU per rank, LOCAL_RANK); rank 0 saves the results and the transfer counters to OUT."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402

FUNCS = ("argmax", "argmin", "nanargmax", "nanargmin")


def programs():
    """(name, source builder, axis): ties everywhere, and the maximum placed in each eighth of a 1-d array in turn (so on
    each rank's part in turn at every world of up to 8 ranks)."""
    r = onp.random.default_rng(11)
    tied = r.integers(-3, 4, size=(48, 20)).astype(onp.float64)
    yield "tied", lambda rb: rb.fromarray(tied), None
    yield "tied_rows", lambda rb: rb.fromarray(tied), 1
    yield "tied_cols", lambda rb: rb.fromarray(tied), 0
    n = 240
    for p in range(8):  # the maximum twice: a tie across the boundary of two eighths
        flat = r.integers(-5, 5, size=n).astype(onp.float64)
        at = p * n // 8 + 3
        flat[at] = 50.0
        flat[min(n - 1, (p + 1) * n // 8)] = 50.0
        flat[(at + 7) % n] = onp.nan
        yield "peak%d" % p, lambda rb, f=flat: rb.fromarray(f), None
    cube = r.integers(-4, 5, size=(6, 40, 5)).astype(onp.int32)
    yield "cube", lambda rb: rb.fromarray(cube), 1
    yield "cube_t", lambda rb: rb.fromarray(cube).T, 2
    yield "bcast", lambda rb: rb.fromarray(cube[:1, :, 0]).broadcast_to((12, 40)), 0
    yield "lazy", lambda rb: rb.fromarray(tied) - rb.fromarray(tied[::-1].copy()), 0


def main():
    import faulthandler

    import _argred_vm
    import _oracle_backend

    faulthandler.dump_traceback_later(int(os.environ.get("RB200_MR_WATCHDOG", "240")), exit=True)
    if (sys.argv[2] if len(sys.argv) > 2 else "oracle") == "oracle":
        _argred_vm.extend_oracle_backend()
        _oracle_backend.install()
    import ramba_b200 as rb
    from ramba_b200 import argreduce, blocks, common
    from ramba_b200.runtime import RT

    if common.num_workers > 1:
        RT.ensure_process_group()
    res = {}
    for name, build, axis in programs():
        A = build(rb)
        rb.sync()
        src = argreduce._source(A)
        cut = axis is None or bool(common.num_workers > 1 and (argreduce._axis_cut(src, axis) or blocks.overlaps_across_ranks(src)))
        for f in FUNCS:
            c0, b0 = RT.collectives, RT.bytes_sent
            r_ = getattr(rb, f)(A, axis=axis)
            c1, b1 = RT.collectives, RT.bytes_sent
            out = onp.asarray(r_.asarray() if isinstance(r_, rb.ndarray) else r_)
            res["%s.%s" % (name, f)] = out
            res["%s.%s.counters" % (name, f)] = onp.array([c1 - c0, b1 - b0, int(cut), max(out.size, 1), int(A.dtype.kind == "f")])
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
