"""rb200_gather / rb200_scatter and the whole `a[idx]` call at 1e9 elements on one GPU, timed with CUDA events.

Index patterns: identity, the fixed-stride permutation (i * 7919) % n and uniform random (seeded).  Byte models:
  * 8 + 2 * itemsize bytes per element (the int64 index read once, the element read once and written once) for every
    pattern;
  * for the random pattern also 8 + 32 + itemsize: every random read pulls a whole 32-byte sector.
The card's name and power limit are read in the same run.  Prints one JSON line per (dtype, pattern)."""
import argparse
import json
import subprocess

import numpy as np
import torch


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return out.strip().splitlines()[0]
    except Exception as ex:  # (the timing does not depend on it)
        return "unknown (%s)" % ex


def time_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    import sys
    import os

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    import ramba_b200 as rb
    from ramba_b200 import _cabi

    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e9)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    n = int(args.n)
    dev = torch.device("cuda", 0)
    name = card()
    for dt in (torch.float64, torch.float32):
        isz = torch.tensor([], dtype=dt).element_size()
        src = torch.rand(n, dtype=dt, device=dev)
        out = torch.empty(n, dtype=dt, device=dev)
        bad = torch.zeros(1, dtype=torch.int64, device=dev)
        view = _cabi.index_view(src.data_ptr(), [n], [1], isz, (src.data_ptr(), src.data_ptr() + n * isz))
        for pat in ("identity", "stride7919", "random"):
            if pat == "identity":
                lin = torch.arange(n, dtype=torch.int64, device=dev)
            elif pat == "stride7919":
                lin = (torch.arange(n, dtype=torch.int64, device=dev) * 7919) % n
            else:
                g = torch.Generator(device=dev)
                g.manual_seed(1234)
                lin = torch.randint(0, n, (n,), generator=g, dtype=torch.int64, device=dev)
            g_ms = time_ms(lambda: _cabi.gather(view, lin.data_ptr(), n, out.data_ptr(), bad.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream), args.reps)
            s_ms = time_ms(lambda: _cabi.scatter(view, lin.data_ptr(), n, out.data_ptr(), bad.data_ptr(),
                                                 torch.cuda.current_stream().cuda_stream), args.reps)
            model = 8 + 2 * isz
            rec = {"card": name, "dtype": str(dt).replace("torch.", ""), "pattern": pat, "n": n, "gather_ms": round(g_ms, 3),
                   "scatter_ms": round(s_ms, 3), "gather_TBps_model_%dB" % model: round(n * model / g_ms / 1e9, 3),
                   "gather_share_of_3.35TBps": round(n * model / g_ms / 1e9 / 3.35, 3),
                   "scatter_TBps_model_%dB" % model: round(n * model / s_ms / 1e9, 3)}
            if pat == "random":
                rec["gather_TBps_model_sector_%dB" % (8 + 32 + isz)] = round(n * (8 + 32 + isz) / g_ms / 1e9, 3)
            print(json.dumps(rec), flush=True)
            del lin
        # the whole a[idx] call (address-stream flush, out-of-range count, gather), identity pattern
        m = n
        A = rb.random.random(m, dtype=np.float64 if dt == torch.float64 else np.float32)
        idx = rb.arange(m)
        A.instantiate()
        idx.instantiate()
        rb.sync()
        call_ms = time_ms(lambda: A[idx], max(2, args.reps // 2))
        print(json.dumps({"card": name, "dtype": str(dt).replace("torch.", ""), "pattern": "identity", "call": "a[idx]", "n": m,
                          "call_ms": round(call_ms, 3)}), flush=True)
        del A, idx, src, out
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
