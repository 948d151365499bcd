#!/usr/bin/env python
"""Generate tests/golden/fancy_golden.npz by running the programs of tests/_fancy_programs.py under the REAL reference
(Python-for-HPC/ramba mounted at /root/reference) in single-worker mode, as make_golden.py does: RAMBA_NON_DIST=1, Ray
replaced by a stub that is never called.  A program the reference cannot run, or whose output differs from NumPy's, is
recorded with the reason in __status__ (and no output of it is stored).

Usage (from the repo root; needs /root/reference and numba):

    python tests/golden/make_fancy_golden.py
"""
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
REF = "/root/reference"

sys.path.insert(0, HERE)
from make_golden import RAY_STUB  # noqa: E402

CHILD = r'''
import json, os, sys
import numpy as onp
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ramba
import _fancy_programs

res, status = {}, {}
for prog in _fancy_programs.PROGRAMS:
    name = prog.__name__
    try:
        got = prog(ramba)
        ramba.sync()
    except Exception as ex:
        status[name] = "reference failed: %s: %s" % (type(ex).__name__, str(ex)[:200])
        continue
    exp = prog(onp)
    diff = [k for k in exp if not (onp.asarray(got[k]).shape == exp[k].shape and onp.array_equal(onp.asarray(got[k]), exp[k]))]
    if diff:
        status[name] = "reference differs from NumPy in %s" % ",".join(diff)
        continue
    for k, v in got.items():
        res["%s__%s" % (name, k)] = onp.asarray(v)
    status[name] = "ok"
res["__status__"] = onp.array(json.dumps(status))
onp.savez_compressed(sys.argv[1], **res)
print(json.dumps(status, indent=1))
'''


def main():
    if not os.path.isdir(REF):
        raise SystemExit("needs the reference at /root/reference (run in the build container)")
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "ray"))
        with open(os.path.join(tmp, "ray", "__init__.py"), "w") as f:
            f.write(RAY_STUB)
        child = os.path.join(tmp, "child.py")
        with open(child, "w") as f:
            f.write("ROOT = %r\n" % ROOT + CHILD)
        env = dict(os.environ)
        env.update({"RAMBA_NON_DIST": "1", "RAMBA_NUM_THREADS": "2", "RAMBA_BIG_DATA": "1",
                    "PYTHONPATH": tmp + ":" + REF, "NUMBA_CACHE_DIR": os.path.join(tmp, "nbcache")})
        out = os.path.join(HERE, "fancy_golden.npz")
        subprocess.check_call([sys.executable, child, out], env=env, cwd=tmp)
        print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
