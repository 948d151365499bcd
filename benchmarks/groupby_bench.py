#!/usr/bin/env python
"""groupby on one GPU: the SUM pass of rb200_group_reduce (CUDA events, median of --reps launches after warm-up) and the
whole calls gb.sum(), gb.mean(), gb.var() and gb - gb.mean() (wall clock to a synchronised result, median of --calls).

Workloads are built on the device (Philox draws of ramba_b200.random); the labels are the day of year (G = 366) or the
season (G = 4) of a 3653-day calendar starting on 2000-01-01, or i % 16 for the flat case.  Bytes = source read + out
written; the fraction is of 3.35 TB/s (H100 SXM HBM3).  Prints one JSON line per workload and the card's name and power
limit, read in the same run; `--out FILE` also writes them as JSON."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import numpy as np  # noqa: E402
import torch  # noqa: E402

PEAK = 3.35e12


def calendar(days=3653):
    d = np.datetime64("2000-01-01") + np.arange(days)
    year_start = d.astype("datetime64[Y]").astype("datetime64[D]")
    doy = (d - year_start).astype(np.int64)                       # 0..365
    month = d.astype("datetime64[M]").astype(np.int64) % 12      # 0..11
    season = np.array([0, 0, 1, 1, 1, 2, 2, 2, 3, 3, 3, 0])[month]  # DJF, MAM, JJA, SON
    return doy, season


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], text=True).strip()
    except Exception as ex:  # noqa: BLE001
        pl = "unknown (%s)" % type(ex).__name__
    return name, pl


def kernel_time(rb, A, gb, reps):
    from ramba_b200 import _cabi, blocks
    from ramba_b200.program import rb_dtype
    from ramba_b200.runtime import RT

    view = blocks.index_view(A)
    table = gb._table(0, A.shape[gb.dim])
    G = gb.num_groups
    n_out = A.size // A.shape[gb.dim] * G
    out = torch.empty(n_out, dtype=torch.float64, device=RT.device)
    nb = _cabi.group_reduce_scratch_bytes(view, gb.dim, G)
    scratch = torch.empty(max(nb, 1), dtype=torch.uint8, device=RT.device)
    plan = _cabi.describe_group_plan(view, gb.dim, G)
    code = rb_dtype(A.dtype)
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        _cabi.group_reduce(view, code, gb.dim, table, _cabi.GROUP_SUM, None, out.data_ptr(), scratch.data_ptr(), stream)
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _cabi.group_reduce(view, code, gb.dim, table, _cabi.GROUP_SUM, None, out.data_ptr(), scratch.data_ptr(), stream)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3)
    t = statistics.median(times)
    nbytes = A.size * A.dtype.itemsize + n_out * 8
    return t, nbytes, plan


def call_time(rb, fn, calls):
    fn()
    rb.sync()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        r = fn()
        r.instantiate()
        rb.sync()
        ts.append(time.perf_counter() - t0)
        del r
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--only", default="")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import ramba_b200 as rb

    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl}))
    doy, season = calendar()
    work = [
        ("rows-doy", (65536, 3653), np.float64, 1, doy, 366),
        ("rows-season", (65536, 3653), np.float64, 1, season, 4),
        ("cols-doy", (3653, 65536), np.float64, 0, doy, 366),
        ("rows-doy-f32", (65536, 3653), np.float32, 1, doy, 366),
        ("cols-doy-f32", (3653, 65536), np.float32, 0, doy, 366),
        ("flat", (1 << 28,), np.float64, 0, np.arange(1 << 28) % 16, 16),
    ]
    results = []
    for wname, shape, dt, dim, labels, G in work:
        if args.only and wname not in args.only.split(","):
            continue
        A = rb.random.default_rng(7).random(shape)
        if dt != np.float64:
            A = A.astype(dt)
        A.instantiate()
        rb.sync()
        gb = A.groupby(dim, labels, G)
        t, nbytes, plan = kernel_time(rb, A, gb, args.reps)
        row = {"name": wname, "shape": list(shape), "dtype": np.dtype(dt).name, "dim": dim, "groups": G, "plan": plan,
               "sum_kernel_ms": round(t * 1e3, 4), "bytes": nbytes, "tb_per_s": round(nbytes / t / 1e12, 4),
               "fraction_of_3.35": round(nbytes / t / PEAK, 4)}
        row["call_sum_ms"] = round(call_time(rb, gb.sum, args.calls) * 1e3, 3)
        row["call_mean_ms"] = round(call_time(rb, gb.mean, args.calls) * 1e3, 3)
        row["call_var_ms"] = round(call_time(rb, gb.var, args.calls) * 1e3, 3)
        row["call_anomaly_ms"] = round(call_time(rb, lambda: gb - gb.mean(), args.calls) * 1e3, 3)
        print(json.dumps(row), flush=True)
        results.append(row)
        del A, gb
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit": pl, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
