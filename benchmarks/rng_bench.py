#!/usr/bin/env python
"""Random fills, the fused Monte-Carlo pi and the host cost of drawing every step, through the public API on cuda:0.

Prints one JSON line with the card's name and power limit read in the same run.  Run it once as it is (plain draws on
the fill kernel, rb200_rng.cu) and once with RB200_NO_RNG=1 (the same draws on the general interpreter):

    python benchmarks/rng_bench.py
    RB200_NO_RNG=1 python benchmarks/rng_bench.py

Fill rates are bytes written over device time (CUDA events around `--reps` back-to-back fills of `--n` elements); a
fill only writes, itemsize bytes per element, so 3.35 TB/s (H100 SXM data sheet) is the bound."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import ramba_b200 as rb  # noqa: E402
from ramba_b200 import _cabi  # noqa: E402

PEAK_BW = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:  # (the measurement still stands with the torch name)
        q = "nvidia-smi unavailable: %s" % ex
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def device_time(fn, reps):
    """Device seconds per call of fn(): CUDA events around `reps` calls after two warm-up calls."""
    for _ in range(2):
        fn()
    rb.sync()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    rb.sync()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e9, help="elements per fill and pairs of the Monte-Carlo pi")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--loop-n", type=int, default=100000, help="elements per step of the draw-every-step loop")
    ap.add_argument("--loop-steps", type=int, default=200)
    args = ap.parse_args()
    n = int(args.n)
    res = {"card": card(), "path": "interpreter" if os.environ.get("RB200_NO_RNG") else "fill_kernel", "n": n}
    rb.random.seed(1)
    keep = []

    def fill(make, itemsize, name):
        def fn():
            keep[:] = [make().instantiate()]  # (run now: a draw nobody reads before the next one replaces it is pruned)
        c0 = _cabi.launch_count()
        t = device_time(fn, args.reps)
        launches = (_cabi.launch_count() - c0) / (args.reps + 2)
        keep[:] = []
        bw = n * itemsize / t
        res[name] = {"ms": round(t * 1e3, 3), "GB_per_s": round(bw / 1e9, 1), "of_3.35TB_per_s": round(bw / PEAK_BW, 3),
                     "launches_per_fill": launches}

    fill(lambda: rb.random.random(n), 8, "uniform_f64")
    fill(lambda: rb.random.random(n, dtype=np.float32), 4, "uniform_f32")
    fill(lambda: rb.random.randn(n), 8, "normal_f64")
    fill(lambda: rb.random.randint(0, 1000, n), 8, "randint_i64")
    rb.sync()
    torch.cuda.empty_cache()

    # fused Monte-Carlo pi: two draws, squares, compare, count - one kernel reading nothing, plus the fold of the partials
    def pi_step():
        return int(((rb.random.rand(n) ** 2 + rb.random.rand(n) ** 2) < 1.0).astype(np.int64).sum())

    pi_step()
    c0 = _cabi.launch_count()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    inside = pi_step()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    launches = _cabi.launch_count() - c0
    est = 4.0 * inside / n
    p = np.pi / 4
    sigma = 4.0 * (p * (1 - p) / n) ** 0.5
    res["monte_carlo_pi"] = {"pairs": n, "seconds": round(dt, 4), "pairs_per_s": round(n / dt / 1e9, 2), "draws_per_s": round(2 * n / dt / 1e9, 2), "unit": "1e9 per s",
                             "launches": launches, "estimate": est, "sigmas_from_pi": round(abs(est - np.pi) / sigma, 2)}

    # host time of a loop that draws every step: a fresh key each step misses the lowering and flush-script memos;
    # re-seeding before each draw repeats the key, and every step is served by the memos
    m = args.loop_n

    def loop(reseed):
        rb.random.seed(3)
        for _ in range(3):
            float((rb.random.rand(m) * 2.0 + 1.0).sum())
        t0 = time.perf_counter()
        for _ in range(args.loop_steps):
            if reseed:
                rb.random.seed(3)
            float((rb.random.rand(m) * 2.0 + 1.0).sum())
        return (time.perf_counter() - t0) / args.loop_steps

    res["draw_every_step"] = {"elements": m, "us_per_step_fresh_key": round(loop(False) * 1e6, 1),
                              "us_per_step_repeated_key": round(loop(True) * 1e6, 1)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
