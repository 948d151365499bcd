#!/usr/bin/env python
"""Generate tests/golden/groupby_golden.npz by running the programs of tests/_groupby_programs.py (the reference's
test_groupby.py restated without xarray, and extra cases) under the REAL reference as build() installs it into
oracle/_ref, in single-worker mode as make_golden.py does: RAMBA_NON_DIST=1, Ray replaced by a stub that is never called.
A program the reference cannot run is recorded with the reason in __status__ (and no output of it is stored).
`nanmean` is not recorded: the reference's NaN test (`value != np.nan`) is always true, so its nanmean is its mean.

Usage (from the repo root, after build(); needs numba):

    python tests/golden/make_groupby_golden.py
"""
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
REF = os.path.join(ROOT, "oracle", "_ref")

sys.path.insert(0, HERE)
from make_golden import RAY_STUB  # noqa: E402

CHILD = r'''
import json, os, sys, warnings
import numpy as onp
sys.path.insert(0, os.path.join(ROOT, "tests"))
warnings.simplefilter("ignore")
import ramba
import _groupby_programs

res, status = {}, {}
for prog in _groupby_programs.PROGRAMS:
    name = prog.__name__
    try:
        with onp.errstate(all="ignore"):
            got = prog(ramba)
        ramba.sync()
    except Exception as ex:
        status[name] = "reference failed: %s: %s" % (type(ex).__name__, str(ex)[:200])
        continue
    for k, v in got.items():
        res["%s__%s" % (name, k)] = onp.asarray(v)
    status[name] = "ok"
res["__status__"] = onp.array(json.dumps(status))
onp.savez_compressed(sys.argv[1], **res)
print(json.dumps(status, indent=1))
'''


def main():
    if not os.path.isdir(os.path.join(REF, "ramba")):
        raise SystemExit("needs the reference installed in oracle/_ref (run build() where the reference is available)")
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
        out = os.path.join(HERE, "groupby_golden.npz")
        subprocess.check_call([sys.executable, child, out], env=env, cwd=tmp)
        print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
