"""Integer-array indexing programs, run in one process (CPU tests, GPU tests) or as one rank of a gloo world:
`_index_worker.py OUT` with RANK / WORLD_SIZE in the environment runs every case through the NumPy restatement of the
kernels (_index_vm) over gloo, `_index_worker.py OUT cuda` through the CUDA library over NCCL (one GPU per rank,
LOCAL_RANK); rank 0 saves the results to OUT."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402

DTYPES = [onp.float64, onp.float32, onp.int64, onp.int32, onp.bool_, onp.uint8, onp.int8, onp.int16, onp.uint16, onp.uint32]


def _data(shape, dtype, seed):
    x = onp.random.default_rng(seed).integers(0, 100, size=shape)
    return (x % 2 == 0) if dtype == onp.bool_ else x.astype(dtype)


def cases():
    """(name, source shape, view of the source, index builder): the builder takes `mk`, which turns a host int array into
    the index array form under test (itself, a list, or a ramba array)."""
    r = onp.random.default_rng(3)
    p1 = r.permutation(23)
    yield "perm1d", (23,), lambda x: x, lambda mk: (mk(p1),)
    yield "neg1d", (23,), lambda x: x, lambda mk: (mk(onp.array([-1, 0, -23, 5, 22], dtype=onp.int32)),)
    yield "dup1d", (23,), lambda x: x, lambda mk: (mk(onp.array([3, 3, 7, 3], dtype=onp.int64)),)
    yield "nested", (6, 7), lambda x: x, lambda mk: (mk(onp.array([[0, 5], [2, 3], [1, 4]], dtype=onp.int16)),)
    yield "adjacent", (5, 6, 7), lambda x: x, lambda mk: (slice(None), mk(onp.array([5, 0, 2])), mk(onp.array([[1], [6]], dtype=onp.uint16)))
    yield "separated", (5, 6, 7), lambda x: x, lambda mk: (mk(onp.array([4, 0, 1])), slice(1, 5), mk(onp.array([6, 2, 0], dtype=onp.int8)))
    yield "int_between", (5, 6, 7), lambda x: x, lambda mk: (mk(onp.array([1, 3])), 2, mk(onp.array([0, 6])))
    yield "int_then_arr", (5, 6, 7), lambda x: x, lambda mk: (slice(None, None, 2), -1, mk(onp.array([[0], [3]])))
    yield "newaxis_ell", (4, 5, 6), lambda x: x, lambda mk: (None, Ellipsis, mk(onp.array([5, 1, 1, 0])))
    yield "sliced_src", (12, 10), lambda x: x[1:11:3, ::-2], lambda mk: (mk(onp.array([3, 0, 2])), mk(onp.array([4, 0, 1])))
    yield "transposed_src", (8, 9), lambda x: x.T, lambda mk: (mk(onp.array([8, 0, 4, 5])), slice(2, 7))
    yield "reversed_src", (30,), lambda x: x[::-1], lambda mk: (mk(onp.array([0, 29, 13])),)
    yield "4d", (3, 4, 5, 6), lambda x: x, lambda mk: (1, slice(None), mk(onp.array([[4], [0]])), mk(onp.array([5, 1, 0])))
    yield "empty_idx", (9,), lambda x: x, lambda mk: (mk(onp.zeros(0, dtype=onp.int64)),)
    yield "size0", (4, 0, 3), lambda x: x, lambda mk: (mk(onp.array([1, 2])),)
    yield "big1d", (5000,), lambda x: x, lambda mk: (mk(((onp.arange(3001) * 7919) % 5000).astype(onp.int64)),)


UNIQUE = {"perm1d", "neg1d", "nested", "adjacent", "separated", "int_between", "int_then_arr", "sliced_src", "transposed_src",
          "reversed_src", "4d", "big1d", "size0", "empty_idx"}


def run_case(rb, name, shape, view, index, dtype, form, local_border=0):
    """(read result, source after a write) through ramba_b200, and the same through NumPy."""
    src = _data(shape, dtype, 11)
    A = rb.fromarray(src, local_border=local_border)
    hi = index(lambda h: h)
    if form == "list":
        ri = index(lambda h: h.tolist())
    elif form == "ramba":
        ri = index(lambda h: rb.fromarray(h))
    else:
        ri = hi
    got_read = view(A)[ri].asarray()
    exp_read = view(src)[hi]
    exp = src.copy()
    vals = _data(exp_read.shape, dtype, 12)
    if name in UNIQUE:
        view(exp)[hi] = vals
        view(A)[ri] = vals
    else:  # duplicate indices: equal values make the result exact
        view(exp)[hi] = vals.reshape(-1)[:1].item() if vals.size else 0
        view(A)[ri] = vals.reshape(-1)[:1].item() if vals.size else 0
    return got_read, exp_read, A.asarray(), exp


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
    for name, shape, view, index in cases():
        for dt in (onp.float64, onp.int16, onp.bool_):
            for form in ("ramba", "list"):
                g, e, ga, ea = run_case(rb, name, shape, view, index, dt, form)
                key = "%s.%s.%s" % (name, onp.dtype(dt).name, form)
                res[key + ".read"], res[key + ".read_exp"] = g, e
                res[key + ".write"], res[key + ".write_exp"] = ga, ea
    # writes through a view into another rank's block; the index array partitioned unlike the source
    a = onp.arange(400, dtype=onp.float64).reshape(20, 20)
    A = rb.fromarray(a)
    Bv = A[::2, 3:]
    c = rb.fromarray(onp.array([[9, 0], [4, 1], [8, 8]]))
    Bv[c, 5] = -1.0
    a[::2, 3:][onp.array([[9, 0], [4, 1], [8, 8]]), 5] = -1.0
    res["view_write"], res["view_write_exp"] = A.asarray(), a
    res["stats"] = onp.array([RT.bytes_sent, RT.collectives])
    # random.choice: one draw, a[integers(0, len(a), size)] of the same generator state
    g = rb.random.default_rng(21)
    pool = onp.arange(100, 137, dtype=onp.float64) * 1.5
    res["choice"] = g.choice(pool, size=(40, 3)).asarray()
    res["choice_int"] = g.choice(50, size=17).asarray()
    rb.sync()
    if common.worker_num == 0:
        onp.savez(sys.argv[1], **res)
    if common.num_workers > 1:  # leave the process group cleanly before the interpreter exits
        import torch.distributed as dist

        dist.barrier()
        dist.destroy_process_group()
    print("ok rank=%d" % common.worker_num)


if __name__ == "__main__":
    main()
