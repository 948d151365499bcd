"""Planning a flush has no side effects (ramba_b200/flush.py::_plan): a flush whose planning fails has launched and
transferred nothing, so the error reaches the caller with the GPU and the other ranks untouched.  At one rank on the
oracle backend, and on a gloo world of 2 with an all-gathered operand (this file is also the worker of that world)."""
import json
import os
import socket
import subprocess
import sys

import numpy as onp
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


class PlanningFailed(Exception):
    pass


def _fail(*a, **k):
    raise PlanningFailed("planning failed")


def _watch_flushes(ramba, RT, set_attr):
    """Wrap the flush entry point: per flush, [launches, collectives, bytes sent] it added, including a flush that raises."""
    deltas = []
    inner = ramba.run_deferred_ops

    def watched(*a, **k):
        c0 = (RT.launches, RT.collectives, RT.bytes_sent)
        try:
            return inner(*a, **k)
        finally:
            deltas.append([RT.launches - c0[0], RT.collectives - c0[1], RT.bytes_sent - c0[2]])

    set_attr(ramba, "run_deferred_ops", watched)
    return deltas


def test_failed_planning_of_an_axis_reduction_launches_nothing(oracle_engine, monkeypatch):
    import ramba_b200 as rb
    from ramba_b200 import flush, ramba
    from ramba_b200.runtime import RT

    x = onp.arange(64 * 48, dtype=onp.float64).reshape(64, 48)
    M = rb.fromarray(x)
    rb.sync()
    flush._plan_cache.clear()
    deltas = _watch_flushes(ramba, RT, monkeypatch.setattr)
    # the combine of stage-1 partials into the partial array is planned after the stage-1 launch
    monkeypatch.setattr(flush, "_combine_program", _fail)
    with pytest.raises(PlanningFailed):
        M.sum(axis=0)
        rb.sync()
    assert deltas == [[0, 0, 0]]


@pytest.mark.timeout(300)
def test_failed_planning_of_a_gathered_operand_transfers_nothing():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    world = 2
    procs = []
    for r in range(world):
        env = dict(os.environ)
        env.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r), "MASTER_ADDR": "127.0.0.1",
                    "MASTER_PORT": str(port), "OMP_NUM_THREADS": "1"})
        procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=240)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, o))
    for rank, (rc, o) in enumerate(outs):
        assert rc == 0, o[-3000:]
        res = json.loads(o.strip().splitlines()[-1])
        assert res["error"] == "planning failed", (rank, res)
        assert res["deltas"] and res["deltas"][-1] == [0, 0, 0], (rank, res)


def _worker():
    """One rank of the gloo world: M + v, where every rank needs the whole of v, which comes by one all-gather; range
    splitting (planned after the pack launch and the all-gather) raises.  Prints what the failed flush added."""
    import faulthandler

    # a rank that dies leaves the other waiting in a collective: dump the stack and exit instead of hanging
    faulthandler.dump_traceback_later(200, exit=True)
    sys.path.insert(0, os.path.join(HERE, ".."))
    sys.path.insert(0, HERE)
    import _oracle_backend

    _oracle_backend.install()
    import ramba_b200 as rb
    from ramba_b200 import flush, ramba, shardview
    from ramba_b200.runtime import RT

    RT.ensure_process_group()
    M = rb.fromarray(onp.arange(240 * 120, dtype=onp.float64).reshape(240, 120))
    v = rb.fromarray(onp.arange(120, dtype=onp.float64))
    rb.sync()
    assert all(int(sv.size[1]) == 120 for sv in M.distribution), "the matrix must be cut into row blocks only"
    flush._plan_cache.clear()
    deltas = _watch_flushes(ramba, RT, setattr)
    shardview.get_range_splits_list = _fail
    error = None
    try:
        (M + v).sum(axis=0)
        rb.sync()
    except PlanningFailed as e:
        error = str(e)
    print(json.dumps({"error": error, "deltas": deltas}))
    sys.stdout.flush()
    import torch.distributed as dist

    dist.barrier()
    faulthandler.cancel_dump_traceback_later()
    dist.destroy_process_group()


if __name__ == "__main__":
    _worker()
