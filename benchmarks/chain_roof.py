#!/usr/bin/env python
"""The headline chain (bench.py config 2: `B = sin(A); C = cos(A); D = B*B + C**2`, float64) on the full and on the lean
instantiation of the 1-D general interpreter, against two roofs for its traffic, one JSON line per arm:

  full       the chain with RB200_NO_LEAN_INTERP=1 (the full interpreter kernel)
  lean       the chain on the lean interpreter kernel
  roof_1r3w  the same traffic without a transcendental, `B = A*1.5; C = A*2.5; D = A*3.5` (must plan as
             kernel=stream, the streaming kernel): the best 1-read / 3-write rate the library reaches
  copy       torch's copy of 8 bytes x n (1 read / 1 write), a reference from outside the library
  lean_walk  the chain with RB200_NO_CTA_PER_TILE=1: the lean kernel on a persistent grid walking tiles b, b+grid, ...
             instead of one CTA per tile (plans without `grid=cta_per_tile`)

What the store form can gain on this traffic was measured with benchmarks/hbm_mix.py (DESIGN §8 item 4): with the
library's layout (2 CTAs/SM walking 2048-element tiles, A staged by bulk copies), 16-byte shuffled stores, bulk
shared -> global stores, contiguous per-CTA tile ranges and 1 or 3 CTAs/SM all write 1R:3W within 0.3 % of plain 8-byte
stores (11.33-11.36 ms for 1e9 float64 elements on an H100 80GB HBM3, 700 W, 1980 MHz).  That is the roof `roof_1r3w`
stands for with the walking grid.  What moved the rate in that probe was the grid: the same work issued as one CTA per
tile, with at most 2 CTAs resident per SM, took 10.84 ms.  The lean interpreter now runs one CTA per tile (`lean`,
against `lean_walk`); the streaming kernel keeps its walk, which was faster for it.

Every arm runs in its own process: the library reads its kill switches once per process, and the arrays of one arm
(A, B, C, D and the previous step's outputs) are gone before the next starts.  Kernel times are CUDA events around
every launch over --steps steps after --warmup steps; the card's name, power limit and SM clock are read in the same
process, after the timed steps.

    python benchmarks/chain_roof.py [--n 1e9] [--steps 30] [--warmup 3] [--arms full,lean,roof_1r3w,copy]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
ARMS = ("full", "lean", "roof_1r3w", "copy", "lean_walk")


def card(dev):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader,nounits", "-i", str(dev)], capture_output=True, text=True)
    if out.returncode != 0:
        return {"card": None}
    name, plim, clk, clk_max = [x.strip() for x in out.stdout.strip().split(",")]
    return {"card": name, "power_limit_w": float(plim), "sm_clock_mhz": int(clk), "sm_clock_max_mhz": int(clk_max)}


def run_arm(arm, n, steps, warmup):
    import torch

    dev = torch.cuda.current_device()
    if arm == "copy":
        src = torch.ones(n, dtype=torch.float64, device="cuda")
        dst = torch.empty_like(src)
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for _ in range(warmup):
            dst.copy_(src)
        for e0, e1 in ev:
            e0.record()
            dst.copy_(src)
            e1.record()
        torch.cuda.synchronize()
        ms = [a.elapsed_time(b) for a, b in ev]
        res = {"plan": "torch copy_", "bytes_per_element": 16, "launches_per_step": 1.0}
    else:
        sys.path.insert(0, ROOT)
        import ramba_b200 as rb
        from ramba_b200 import _cabi
        from ramba_b200.runtime import RT

        A = rb.arange(n) / 1000.0
        rb.sync()
        out = []

        def step():
            if arm == "roof_1r3w":
                B, C, D = A * 1.5, A * 2.5, A * 3.5
            else:
                B = rb.sin(A)
                C = rb.cos(A)
                D = B * B + C ** 2
            rb.sync()
            out[:] = [B, C, D]

        be = RT.be()
        run, plans = be.run, []

        def record(fop, stream=None):
            plans.append(_cabi.describe_plan(fop))
            return run(fop, stream)

        be.run = record
        step()
        be.run = run
        for _ in range(warmup):
            step()
        RT.profile_events = []
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
        events, RT.profile_events = RT.profile_events, None
        ms = [a.elapsed_time(b) for a, b, _ in events]
        res = {"plan": plans, "bytes_per_element": 32, "launches_per_step": len(ms) / steps}
        assert all(("grid=cta_per_tile" in p) == (arm == "lean") for p in plans), plans
        if arm == "roof_1r3w":
            assert all(p.startswith("kernel=stream ") for p in plans), plans
        else:
            assert all(p.startswith("kernel=general_interpreter form=elementwise") for p in plans), plans
            assert all(("variant=lean" in p) == (arm != "full") for p in plans), plans
            d = out[2][0:4096].asarray()
            import numpy as np

            assert float(np.max(np.abs(d - 1.0))) <= 4 * np.finfo(np.float64).eps
    kernel_ms = sum(ms) / len(ms)
    res.update({"arm": arm, "n": n, "steps": steps, "kernel_ms": kernel_ms, "kernel_ms_min": min(ms), "kernel_ms_max": max(ms),
                "gbps": res["bytes_per_element"] * n / kernel_ms / 1e6})
    res.update(card(dev))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e9)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--arms", default=",".join(ARMS))
    ap.add_argument("--arm", help=argparse.SUPPRESS)  # one arm in this process
    args = ap.parse_args()
    assert args.steps >= 20, "time at least 20 launches"
    if args.arm:
        print(json.dumps(run_arm(args.arm, int(args.n), args.steps, args.warmup)), flush=True)
        return
    for arm in args.arms.split(","):
        assert arm in ARMS, arm
        env = dict(os.environ)
        env.pop("RB200_NO_LEAN_INTERP", None)
        env.pop("RB200_NO_CTA_PER_TILE", None)
        if arm == "full":
            env["RB200_NO_LEAN_INTERP"] = "1"
        if arm == "lean_walk":
            env["RB200_NO_CTA_PER_TILE"] = "1"
        cmd = [sys.executable, os.path.abspath(__file__), "--arm", arm, "--n", str(args.n), "--steps", str(args.steps), "--warmup", str(args.warmup)]
        subprocess.run(cmd, env=env, check=True)


if __name__ == "__main__":
    main()
