"""Process-wide configuration: environment flags and the worker (= rank = GPU) identity.

Mirrors the flag names of the reference (ramba/common.py:30-211, README table) so that a user's
environment keeps working; flags that only make sense for Ray/MPI/Numba are accepted and ignored.

Execution model: SPMD, one process per GPU, every rank runs the same driver program and owns
division `rank` of every array (the reference's SPMD-under-MPI mode, ramba/ramba.py:3986-3993,
10683-10690).  `num_workers` is the launcher's WORLD_SIZE (1 without a launcher).
"""
import os
import sys
import time

distribute_min_size = 100  # ramba/common.py:26
NUM_WORKERS_FOR_BCAST = 100


def _env_int(name, default=0):
    v = os.environ.get(name)
    if v is None:
        return default
    try:
        return int(v)
    except ValueError:
        return default


ndebug = _env_int("RAMBA_DEBUG", 0)
ntiming = _env_int("RAMBA_TIMING", 0)
debug_showcode = _env_int("RAMBA_SHOW_CODE", 0) != 0
reshape_forwarding = _env_int("RAMBA_RESHAPE_COPY", 0) != 0  # reshape() calls forward to reshape_copy (ramba/common.py:141-146)
ramba_big_data = True  # indices are always int64 here (RAMBA_BIG_DATA, ramba/shardview_array.py:24-28)

# worker identity: torchrun exports RANK / WORLD_SIZE / LOCAL_RANK
worker_num = _env_int("RANK", 0)
num_workers = _env_int("WORLD_SIZE", 1)
local_rank = _env_int("LOCAL_RANK", worker_num)
num_nodes = 1  # one 8xH100 box: every peer is one NVSwitch hop away


def set_world(rank, world):
    """Re-point the process at a different (rank, world) — used by tests that emulate workers."""
    global worker_num, num_workers
    worker_num = int(rank)
    num_workers = int(world)


def do_not_distribute(size):
    """Arrays with fewer than distribute_min_size elements live wholly on worker 0
    (ramba/common.py:217-218)."""
    n = 1
    for s in size:
        n *= int(s)
    return n < distribute_min_size


def dprint(level, *args):
    if ndebug >= level:
        print(*args)
        sys.stdout.flush()


def tprint(level, *args):
    if ntiming >= level:
        print(*args)
        sys.stdout.flush()


timer = time.perf_counter

# ---- timing registry (ramba/ramba.py:923-1020: add_time / add_sub_time / get_timing)
time_dict = {}
sub_time_dict = {}


def add_time(name, val):
    t = time_dict.setdefault(name, [0, 0.0])
    t[0] += 1
    t[1] += val


def add_sub_time(name, sub, val):
    t = sub_time_dict.setdefault(name, {}).setdefault(sub, [0, 0.0])
    t[0] += 1
    t[1] += val


def reset_timing():
    time_dict.clear()
    sub_time_dict.clear()


def get_timing(details=False):
    if details:
        return {k: (tuple(v), {s: tuple(x) for s, x in sub_time_dict.get(k, {}).items()}) for k, v in time_dict.items()}
    return {k: v[1] for k, v in time_dict.items()}


def get_timing_str(details=False):
    out = []
    for k, v in time_dict.items():
        out.append("%s: %.6fs (%d)" % (k, v[1], v[0]))
        if details:
            for s, x in sub_time_dict.get(k, {}).items():
                out.append("    %s: %.6fs (%d)" % (s, x[1], x[0]))
    return "\n".join(out)
