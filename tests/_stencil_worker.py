"""The stencil cases of test_stencil_semantics run as one rank of a world: `_stencil_worker.py OUT` with RANK / WORLD_SIZE
in the environment runs them through the oracle backend over gloo.  Rank 0 saves every output and the blocks each rank
held of the case's first input to OUT; every rank builds the same input values."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402

import test_stencil_semantics as T  # noqa: E402


def main():
    import faulthandler

    import _oracle_backend

    faulthandler.dump_traceback_later(int(os.environ.get("RB200_MR_WATCHDOG", "600")), exit=True)
    _oracle_backend.install()
    import ramba_b200 as rb
    from ramba_b200 import common
    from ramba_b200.runtime import RT

    if common.num_workers > 1:
        RT.ensure_process_group()
    res = {}
    for name in T.WORLD_CASES:
        c = next(c for c in T.CASES if c.name == name)
        X = {k: rb.fromarray(v, **(c.border or {})) for k, v in c.inputs.items()}
        first = X[next(iter(c.inputs))]
        res[name + ".blocks"] = onp.array([[int(s) for s in sv.start] + [int(s) for s in sv.size] for sv in first.distribution], dtype=onp.int64)
        for i, o in enumerate(c.run(rb, X)):
            res["%s.%d" % (name, i)] = onp.asarray(o.asarray())
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
