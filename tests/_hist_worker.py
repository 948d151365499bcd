"""histogram / bincount / searchsorted / digitize programs, run as one rank of a world: `_hist_worker.py OUT` with RANK /
WORLD_SIZE in the environment runs them through the NumPy restatement of the kernels (_hist_vm) over gloo,
`_hist_worker.py OUT cuda` through the CUDA library over NCCL (one GPU per rank, LOCAL_RANK); rank 0 saves the results
and the transfer counters to OUT."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402


def data():
    r = onp.random.default_rng(11)
    x = r.standard_normal((40, 37))
    x[r.random(x.shape) < 0.05] = 0.25  # values on an edge of bins=8, range=(-2, 2)
    lab = r.integers(0, 30, 700)
    lab[::97] = 0
    w = r.standard_normal(700) * 1e3
    return x, lab, w


def programs():
    """(name, call(rb, host arrays) -> tuple of results, collectives at several ranks: None when the engine's min and
    max reductions come first)."""
    yield "hist_range", lambda rb, x, lab, w: rb.histogram(rb.fromarray(x), bins=8, range=(-2, 2)), 1
    yield "hist_auto", lambda rb, x, lab, w: rb.histogram(rb.fromarray(x), bins=13), None
    yield "hist_edges", lambda rb, x, lab, w: rb.histogram(rb.fromarray(x).T, bins=[-3, -1, 0, 0.25, 2, 9]), 1
    yield "hist_weighted", lambda rb, x, lab, w: rb.histogram(rb.fromarray(lab * 0.5), bins=10, range=(0, 15), weights=rb.fromarray(w)), 1
    yield "bincount", lambda rb, x, lab, w: (rb.bincount(rb.fromarray(lab)),), None
    yield "bincount_w", lambda rb, x, lab, w: (rb.bincount(rb.fromarray(lab), weights=rb.fromarray(w), minlength=40),), None
    yield "search_host", lambda rb, x, lab, w: (rb.searchsorted(onp.sort(x[0]), rb.fromarray(x), side="right"),), 0
    yield "search_ramba", lambda rb, x, lab, w: (rb.searchsorted(rb.fromarray(onp.sort(x[1])), rb.fromarray(x)[::2]),), 1
    yield "digitize", lambda rb, x, lab, w: (rb.digitize(rb.fromarray(x), onp.array([2.0, 1.0, 0.0, -1.0]), right=True),), 0


def main():
    import faulthandler

    import _hist_vm
    import _oracle_backend

    faulthandler.dump_traceback_later(int(os.environ.get("RB200_MR_WATCHDOG", "240")), exit=True)
    if (sys.argv[2] if len(sys.argv) > 2 else "oracle") == "oracle":
        _hist_vm.extend_oracle_backend()
        _oracle_backend.install()
    import ramba_b200 as rb
    from ramba_b200 import common
    from ramba_b200.runtime import RT

    if common.num_workers > 1:
        RT.ensure_process_group()
    x, lab, w = data()
    res = {}
    for name, call, _ in programs():
        rb.sync()
        c0, b0 = RT.collectives, RT.bytes_sent
        outs = call(rb, x, lab, w)
        rb.sync()
        c1, b1 = RT.collectives, RT.bytes_sent
        for i, o in enumerate(outs):
            res["%s.%d" % (name, i)] = o.asarray()
        res["%s.counters" % name] = onp.array([c1 - c0, b1 - b0])
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
