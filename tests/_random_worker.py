"""Worker process of the random-draw tests.  `_random_worker.py OUT [oracle]`: RANK / WORLD_SIZE come from the environment,
collectives run over gloo, op lists through the NumPy oracle extended by PHILOX (_philox_vm).  `_random_worker.py OUT gpu`:
one process on cuda:0.  Every program runs twice (the second run replays the memoised flush scripts); rank 0 saves what
both runs produced to OUT."""
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

import ramba_b200 as rb  # noqa: E402
from ramba_b200 import common  # noqa: E402
from ramba_b200.runtime import RT  # noqa: E402

# GPU mode: every form over ragged 1-D, 2-D and 3-D shapes (the fill kernel, or the interpreter with RB200_NO_RNG=1)
GPU_SHAPES = [(1000003,), (517, 301), (7, 33, 65)]


def gpu_forms(out):
    for si, shape in enumerate(GPU_SHAPES):
        rb.random.seed(100 + si)
        out["u64_%d" % si] = rb.random.random(shape).asarray()
        out["u32_%d" % si] = rb.random.random(shape, dtype=onp.float32).asarray()
        out["n64_%d" % si] = rb.random.randn(*shape).asarray()
        out["int_%d" % si] = rb.random.randint(-7, 1000, shape).asarray()
        out["aff_%d" % si] = rb.random.normal(3.0, 0.5, shape).asarray()


def plain(out):
    """1-D, 2-D and 3-D draws of every form, below and above distribute_min_size, with ragged divisions."""
    rb.random.seed(7)
    out["u1"] = rb.random.random(1001).asarray()
    out["small"] = rb.random.rand(5).asarray()
    out["u32"] = rb.random.random((37, 53), dtype=onp.float32).asarray()
    out["n2"] = rb.random.normal(2.0, 3.0, (64, 33)).asarray()
    out["i3"] = rb.random.randint(3, 17, (11, 7, 5)).asarray()
    out["uni"] = rb.random.uniform(-1.0, 2.0, 999).asarray()
    out["g"] = rb.random.default_rng(11).integers(0, 1 << 40, (9, 301)).asarray()
    out["rs"] = rb.random.RandomState(1337).normal(loc=5.0, size=(1000, 10)).asarray()


def views(out):
    """Draws assigned into slices and transposed views."""
    rb.random.seed(8)
    a = rb.zeros((40, 30))
    a[5:25, 3:13] = rb.random.rand(20, 10)
    b = rb.zeros((30, 40))
    bt = b.T
    bt[:, :] = rb.random.randn(40, 30)
    c = rb.zeros(500, dtype=onp.int64)
    c[100:400] = rb.random.randint(-50, 50, 300)
    out["a"], out["b"], out["c"] = a.asarray(), b.asarray(), c.asarray()


def fused(out):
    """Draws consumed in fused arithmetic and reductions, without being stored."""
    rb.random.seed(9)
    n = 5000
    x = rb.random.rand(n)
    y = rb.random.rand(n)
    out["inside"] = onp.array(int(((x * x + y * y) < 1.0).astype(onp.int64).sum()))
    out["colcount"] = ((rb.random.randn(60, 50) * 2.0 + 1.0) > 0.0).astype(onp.int64).sum(axis=0).asarray()
    out["count"] = onp.array(int((rb.random.uniform(1.0, 2.0, (13, 17, 19)) < 1.5).astype(onp.int64).sum()))
    # float sums: the draws are the same on every partition, the order of the additions is not
    out["fsum_cols"] = (rb.random.randn(60, 50) * 2.0 + 1.0).sum(axis=0).asarray()
    out["fsum"] = onp.array(float((rb.random.uniform(1.0, 2.0, (13, 17, 19)) * 0.5).sum()))
    out["mixed"] = (rb.random.rand(4000) + rb.random.random(4000, dtype=onp.float32)).asarray()


PROGRAMS = [plain, views, fused]


def main():
    import faulthandler

    faulthandler.dump_traceback_later(int(os.environ.get("RB200_MR_WATCHDOG", "240")), exit=True)
    if common.num_workers > 1:
        RT.ensure_process_group()
    res = {}
    for run in range(2):
        for p in (PROGRAMS if MODE == "oracle" else [gpu_forms]):
            out = {}
            p(out)
            for k, v in out.items():
                res["%s.%s.%d" % (p.__name__, k, run)] = v
    rb.sync()
    if common.worker_num == 0:
        onp.savez(sys.argv[1], **res)
    if common.num_workers > 1:  # leave the process group cleanly before the interpreter exits
        import torch.distributed as dist

        dist.barrier()
        dist.destroy_process_group()
    print("ok rank=%d launches=%d" % (common.worker_num, RT.launches))


if __name__ == "__main__":
    main()
