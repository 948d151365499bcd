"""RT.bytes_sent / RT.collectives (bench.py's bytes_sent_per_rank_per_step and collectives_per_step) follow one counting
rule for every operation that talks to other ranks, and a repeated flush counts what its first run counted: gloo worlds
2 and 3, each rank checked against the rule worked out from the shapes and partitions (tests/_counters_worker.py)."""
import json
import os
import socket
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = ["halo", "gathered", "reshape_copy", "getitem", "setitem", "cumsum", "global_sum", "axis_sum", "asarray", "unseeded_draw"]


@pytest.fixture(params=[2, 3], ids=lambda world: "world%d" % world)
def counted(request):
    """One run of the worker on a gloo world: per rank, {case: {"first", "again", "expected", "planned"}}."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    world = request.param
    procs = []
    for r in range(world):
        env = dict(os.environ)
        env.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r), "MASTER_ADDR": "127.0.0.1",
                    "MASTER_PORT": str(port), "OMP_NUM_THREADS": "1"})
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_counters_worker.py")], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=240)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, o))
    for rc, o in outs:
        assert rc == 0, o[-3000:]
    return [json.loads(o.strip().splitlines()[-1]) for _, o in outs]


@pytest.mark.timeout(300)
def test_every_transfer_is_counted_by_one_rule(counted):
    wrong = []
    for rank, res in enumerate(counted):
        assert sorted(res) == sorted(CASES), rank
        for case, r in res.items():
            if r["first"] != r["expected"]:
                wrong.append("rank %d %s: counted %s, the rule gives %s" % (rank, case, r["first"], r["expected"]))
            if r["again"] != r["first"]:
                wrong.append("rank %d %s: counted %s the second time, %s the first" % (rank, case, r["again"], r["first"]))
        # the flushes of the halo exchange and of the all-gathered operand were planned the first time only: the second
        # time they ran their memoised scripts
        for case in ("halo", "gathered"):
            assert res[case]["planned"][0] > 0 and res[case]["planned"][1] == 0, (rank, case, res)
    assert not wrong, "\n".join(wrong)
