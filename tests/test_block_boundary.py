"""The boundary between the array code and this rank's blocks, kernels and buffers.

Structure (read from the package's source): the runtime is the only module that calls the backend or counts launches;
blocks are created outside a flush by blocks.py only; buffers are held by RT.hold only; the DAG's internals stay in
ramba.py.  Behaviour: an array read before it is ever written, and then written in the same fused op as a statement over
a different partition of its shape, keeps the partition its block was made at (gloo world 2)."""
import ast
import os
import re
import socket
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(HERE, "..", "ramba_b200")


def _modules():
    for name in sorted(os.listdir(PKG)):
        if name.endswith(".py"):
            with open(os.path.join(PKG, name)) as f:
                yield name, ast.parse(f.read(), name)


def _sites(pred):
    """{module: [line]} of the nodes for which pred(node) holds."""
    hits = {}
    for name, tree in _modules():
        for node in ast.walk(tree):
            if pred(node):
                hits.setdefault(name, []).append(node.lineno)
    return hits


def _calls(attr):
    return lambda n: isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and n.func.attr == attr


def _assigns(attr):
    def pred(n):
        targets = n.targets if isinstance(n, ast.Assign) else [n.target] if isinstance(n, ast.AugAssign) else []
        return any(isinstance(t, ast.Attribute) and t.attr == attr for t in targets)

    return pred


def test_only_the_runtime_calls_the_backend_and_counts_launches():
    assert set(_sites(_calls("be"))) <= {"runtime.py"}, _sites(_calls("be"))
    assert set(_sites(_assigns("launches"))) == {"runtime.py"}, _sites(_assigns("launches"))


def test_only_the_flush_and_blocks_create_shards():
    assert set(_sites(_calls("create_array"))) == {"flush.py", "blocks.py"}, _sites(_calls("create_array"))


def test_only_blocks_and_the_fuser_fix_a_partition():
    """remote_constructed is set by blocks.block and by the fuser's _finish (and initialised by bdarray)."""
    where = set()
    for name, tree in _modules():
        for fn in ast.walk(tree):
            if isinstance(fn, (ast.FunctionDef, ast.AsyncFunctionDef)):
                if any(_assigns("remote_constructed")(n) for n in ast.walk(fn)):
                    where.add((name, fn.name))
    assert where == {("blocks.py", "block"), ("ramba.py", "_finish"), ("ramba.py", "__init__")}, where


def test_buffers_are_held_one_way():
    """No keepalive / keepalive_* attribute: RT.hold is the one way to keep buffers alive past a call."""
    old = re.compile(r"keepalive(_\w+)?$")
    hits = _sites(lambda n: isinstance(n, ast.Attribute) and old.match(n.attr))
    assert not hits, hits


def test_the_dag_internals_stay_in_ramba():
    def pred(n):
        if not (isinstance(n, ast.Attribute) and n.attr in ("readers", "last_writer", "_run")):
            return False
        v = n.value
        return (isinstance(v, ast.Name) and v.id == "DAG") or (isinstance(v, ast.Attribute) and v.attr == "DAG")

    assert set(_sites(pred)) <= {"ramba.py"}, _sites(pred)


_READ_THEN_WRITE = r"""
import sys
sys.path[:0] = [%r, %r]
import numpy as onp
import _oracle_backend
_oracle_backend.install()
import ramba_b200 as rb
from ramba_b200 import common, shardview
from ramba_b200.runtime import RT

RT.ensure_process_group()
w = common.worker_num
n = 100
x = onp.arange(n, dtype=onp.int64)
split = [shardview.shardview(onp.array([30]), onp.array([0])), shardview.shardview(onp.array([70]), onp.array([30]))]
b = rb.fromarray(x, distribution=split)     # not the default partition of its shape (50 / 50)
a = rb.empty(n, dtype=onp.int64)
rb.local_block_to_host(a)                   # read before any write: this rank's block of the default partition
b += 1                                      # pending, over b's partition
a *= 0                                      # same shape: may share b's fused op only if a's partition can still move
a += b
got = rb.local_block_to_host(a)
sv = a.distribution[w]
assert RT.shards[a.gid].shape == (int(sv.size[0]),), (w, RT.shards[a.gid].shape, sv.size)  # the block fits the partition
exp = (x + 1)[int(sv.start[0]):int(sv.start[0]) + int(sv.size[0])]
assert onp.array_equal(got, exp), (w, got, exp)
import torch.distributed as dist
dist.barrier()
dist.destroy_process_group()
print("ok")
"""


def test_a_block_read_before_its_first_write_keeps_its_partition():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    code = _READ_THEN_WRITE % (os.path.join(HERE, ".."), HERE)
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                   OMP_NUM_THREADS="1")
        procs.append(subprocess.Popen([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                      text=True))
    deadline = time.time() + 240
    while any(p.poll() is None for p in procs):
        if any(p.returncode not in (None, 0) for p in procs) or time.time() > deadline:
            break  # (a rank that failed leaves its peer waiting in a collective)
        time.sleep(0.1)
    for p in procs:
        if p.poll() is None:
            p.kill()
    outs = [p.communicate()[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and o.strip().endswith("ok"), "rank %d:\n%s" % (r, o[-3000:])
