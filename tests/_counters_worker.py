"""Worker process of tests/test_transfer_counters.py (RANK / WORLD_SIZE from the environment, gloo between the ranks, op
lists through the oracle).  Runs every operation that talks to other ranks once, then again so that its flushes run
their memoised scripts, and records how much RT.bytes_sent / RT.collectives grew each time next to what the counting
rule of DESIGN.md §4 gives for the shapes and partitions involved:

  grouped send / receive: the bytes of every send, no collective;  all-gather: 1 collective, bytes of this rank's part
  times W-1;  all-reduce: 1 collective, bytes of the tensor;  broadcast: 1 collective and, on the source rank only, bytes
  of the tensor times W-1.

Prints one JSON line: {case: {"first": [bytes, collectives], "again": [...], "expected": [...], "planned": [flushes
planned the first time, the second time]}}."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import numpy as onp  # noqa: E402

import _oracle_backend  # noqa: E402

_oracle_backend.install()

import ramba_b200 as rb  # noqa: E402
from ramba_b200 import common, flush  # noqa: E402
from ramba_b200.runtime import RT  # noqa: E402

w, W = common.worker_num, common.num_workers
F64 = 8  # bytes of one float64 / int64 element (and of the reductions' accumulators)


def owner(nd):
    """Which rank holds every element of whole array nd, from its partition."""
    own = onp.full(nd.shape, -1)
    for r, sv in enumerate(nd.distribution):
        own[tuple(slice(int(a), int(a) + int(n)) for a, n in zip(sv.start, sv.size))] = r
    return own


def part_elems(nd, r):
    return int(onp.prod([int(n) for n in nd.distribution[r].size]))


# Every case sets up its arrays and returns run(): the operation, then the (bytes, collectives) the rule expects for it.
def halo():
    n = 120
    U = rb.fromarray(onp.arange(n, dtype=onp.float64))
    V = rb.zeros(n)
    rb.sync()

    def run():
        V[1:-1] = U[:-2] + U[2:]
        rb.sync()
        # iteration i runs where V[i] lives and reads U[i-1], U[i+1]: each element of mine a peer reads is one send
        ou, ov = owner(U), owner(V)
        sent = sum(1 for i in range(1, n - 1) for j in (i - 1, i + 1) if ou[j] == w and ov[i] != w)
        return F64 * sent, 0

    return run


def gathered():
    # config 5 scaled down: a vector cut into chunks, added to every row of a matrix cut into row blocks; every rank
    # needs the whole vector, which comes by one all-gather
    M = rb.fromarray(onp.arange(240 * 120, dtype=onp.float64).reshape(240, 120))
    v = rb.fromarray(onp.arange(120, dtype=onp.float64))
    rb.sync()
    assert all(int(sv.size[1]) == 120 for sv in M.distribution), "the matrix must be cut into row blocks only"

    def run():
        R = M + v
        rb.sync()
        assert R.shape == (240, 120)
        return F64 * part_elems(v, w) * (W - 1), 1

    return run


def reshape_copy():
    a = rb.fromarray(onp.arange(120, dtype=onp.float64).reshape(12, 10))
    rb.sync()

    def run():
        out = rb.reshape_copy(a, (10, 12))
        rb.sync()
        # every element of my source block that lands in another rank's destination block is sent once
        src, dst = owner(a).ravel(), owner(out).ravel()
        return F64 * int(((src == w) & (dst != w)).sum()), 0

    return run


_IDX = (onp.arange(120) * 37 + 11) % 120


def _requests(a, lin_like):
    """m[p][q]: requests of rank p (its block of the index) for elements rank q holds."""
    oa, ol = owner(a), owner(lin_like)
    m = onp.zeros((W, W), dtype=onp.int64)
    for k, i in enumerate(_IDX):
        m[ol[k], oa[i]] += 1
    return m


def _index_common():
    # the count of out-of-range indices (a global sum: one 8-byte all-reduce) and the request counts (an all-gather of W
    # int64 per rank)
    return F64 + F64 * W * (W - 1), 2


def getitem():
    a = rb.fromarray(onp.arange(120, dtype=onp.float64) * 0.5)
    lin_like = rb.empty(_IDX.shape, dtype=onp.int64)
    rb.sync()

    def run():
        r = a[_IDX]
        rb.sync()
        m = _requests(a, lin_like)
        b, c = _index_common()
        others = [q for q in range(W) if q != w]
        # requests out (int64 offsets), replies out (float64 values)
        return b + sum(F64 * int(m[w][q]) for q in others) + sum(F64 * int(m[q][w]) for q in others), c

    return run


def setitem():
    a = rb.fromarray(onp.arange(120, dtype=onp.float64) * 0.5)
    lin_like = rb.empty(_IDX.shape, dtype=onp.int64)
    rb.sync()

    def run():
        a[_IDX] = 7.0
        rb.sync()
        m = _requests(a, lin_like)
        b, c = _index_common()
        # requests and their values out, together
        return b + sum((F64 + F64) * int(m[w][q]) for q in range(W) if q != w), c

    return run


def cumsum():
    x = rb.fromarray(onp.arange(120, dtype=onp.float64))
    rb.sync()

    def run():
        r = rb.cumsum(x)
        rb.sync()
        assert r.shape == (120,)
        return F64 * 1 * (W - 1), 1  # one total per block (one column), all-gathered

    return run


def global_sum():
    x = rb.fromarray(onp.arange(120, dtype=onp.float64))
    rb.sync()

    def run():
        assert float(x.sum()) == float(onp.arange(120).sum())
        return F64, 1  # one partial per rank, all-reduced

    return run


def axis_sum():
    M = rb.fromarray(onp.arange(240 * 120, dtype=onp.float64).reshape(240, 120))
    rb.sync()

    def run():
        r = M.sum(axis=0)
        rb.sync()
        assert r.shape == (120,)
        return F64 * 120, 1  # the partial row of every rank, all-reduced

    return run


def asarray():
    x = rb.fromarray(onp.arange(120, dtype=onp.float64))
    rb.sync()

    def run():
        assert onp.array_equal(x.asarray(), onp.arange(120))
        parts = [r for r in range(W) if part_elems(x, r)]
        return F64 * part_elems(x, w) * (W - 1), len(parts)  # every part broadcast from its owner

    return run


def unseeded_draw():
    def run():
        d = rb.random.default_rng().random(120)
        rb.sync()
        assert d.shape == (120,)
        return (F64 * (W - 1) if w == 0 else 0), 1  # rank 0's seed, broadcast

    return run


CASES = [halo, gathered, reshape_copy, getitem, setitem, cumsum, global_sum, axis_sum, asarray, unseeded_draw]


def main():
    import faulthandler

    # a rank that dies leaves the others waiting in a collective: dump the stack and exit instead of hanging
    faulthandler.dump_traceback_later(int(os.environ.get("RB200_MR_WATCHDOG", "240")), exit=True)
    RT.ensure_process_group()
    flush._VERIFY_PLAN_CACHE = False  # the second runs must not plan the flushes again (verification mode does)
    planned = [0]
    plan = flush._plan

    def counted(*a, **k):
        planned[0] += 1
        return plan(*a, **k)

    flush._plan = counted
    out = {}
    for case in CASES:
        run = case()
        got = []
        plans = []
        for _ in range(2):
            planned[0] = 0
            b0, c0 = RT.bytes_sent, RT.collectives
            exp = run()
            got.append([RT.bytes_sent - b0, RT.collectives - c0])
            plans.append(planned[0])
        out[case.__name__] = {"first": got[0], "again": got[1], "expected": list(exp), "planned": plans}
    print(json.dumps(out))
    sys.stdout.flush()
    import torch.distributed as dist

    dist.barrier()
    faulthandler.cancel_dump_traceback_later()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
