"""median / percentile / quantile programs, run as one rank of a world: `_quantile_worker.py OUT` with RANK / WORLD_SIZE in
the environment runs them through the NumPy restatement of the kernels (_select_vm) over gloo, `_quantile_worker.py OUT
cuda` through the CUDA library over NCCL (one GPU per rank, LOCAL_RANK); rank 0 saves the results and the transfer
counters to OUT."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402


def data():
    r = onp.random.default_rng(13)
    x = r.standard_normal((40, 37))
    x[r.random(x.shape) < 0.05] = onp.nan
    x[3, :] = onp.nan  # an all-NaN row
    return x


def programs():
    """(name, call(rb, x) -> result, reduced axis (None: every axis), targets per segment)."""
    yield "median_all", lambda rb, x: rb.median(rb.fromarray(onp.nan_to_num(x))), None, 2
    yield "nanmedian_all", lambda rb, x: rb.nanmedian(rb.fromarray(x)), None, 2
    yield "pct_all", lambda rb, x: rb.percentile(rb.fromarray(onp.nan_to_num(x)), [1, 25, 50, 75, 99]), None, 10
    yield "median_ax1", lambda rb, x: rb.median(rb.fromarray(x), axis=1), 1, 2
    yield "nanquantile_ax1", lambda rb, x: rb.nanquantile(rb.fromarray(x), [0.1, 0.9], axis=1, keepdims=True), 1, 4
    yield "median_ax0", lambda rb, x: rb.median(rb.fromarray(onp.nan_to_num(x)), axis=0), 0, 2
    yield "nanpct_ax0", lambda rb, x: rb.nanpercentile(rb.fromarray(x), 30, axis=0), 0, 2


def global_rows(name, x):
    """(global segments, passes, digit, nan all-reduces) of a program that all-reduces its counts."""
    K = {n: k for n, _, _, k in programs()}[name]
    ax = {n: a for n, _, a, _ in programs()}[name]
    GS = 1 if ax is None else x.shape[1 - ax]
    digit = 11 if GS == 1 and K <= 12 else 8
    return GS, -(-64 // digit), digit, 1


def main():
    import faulthandler
    import warnings

    import _oracle_backend
    import _select_vm

    faulthandler.dump_traceback_later(int(os.environ.get("RB200_MR_WATCHDOG", "240")), exit=True)
    if (sys.argv[2] if len(sys.argv) > 2 else "oracle") == "oracle":
        _select_vm.extend_oracle_backend()
        _oracle_backend.install()
    import ramba_b200 as rb
    from ramba_b200 import common
    from ramba_b200.runtime import RT

    if common.num_workers > 1:
        RT.ensure_process_group()
    x = data()
    res = {}
    X = rb.fromarray(x)
    for name, call, ax, _ in programs():
        # the axis is cut when some rank's part does not span it (every axis at once: always, at several ranks)
        cut = common.num_workers > 1 and (ax is None or any(int(sv.start[ax]) != 0 or int(sv.size[ax]) != x.shape[ax] for sv in X.distribution
                                                            if int(sv.size.prod()) > 0))
        res["%s.cut" % name] = onp.array(cut)
        rb.sync()
        c0, b0 = RT.collectives, RT.bytes_sent
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out = call(rb, x)
        rb.sync()
        c1, b1 = RT.collectives, RT.bytes_sent
        res[name] = out.asarray() if hasattr(out, "asarray") else onp.asarray(out)
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
