#!/usr/bin/env python
"""HBM rate of write-heavy float64 streams on one GPU: the library's store form against candidate forms, one JSON line
per arm.

The probe kernels (ramba_b200/csrc/probe/rb200_hbm_probe.cu, `make -C ramba_b200/csrc probe`, a shared object of
their own) compute `out_j = A * s_j` for one or three outputs with the layout of the library's 1-D kernels (256
threads, element k of thread t at tile*2048 + k*256 + t, A staged by bulk copies into a ring).  Arms:

  copy, fill           torch `copy_` (1 read / 1 write) and `fill_` (0 / 1): references from outside the library
  lib_1r3w_d2 / _d6    the library's form: 8-byte stores, round-robin tile walk, 2 CTAs/SM; input ring of 2 stages
                       (the lean interpreter) or 6 (the streaming kernel on one staged view)
  lib_1r1w             the same form with one output
  shfl16               (a) warp-pair shuffle to 16-byte stores
  bulk                 (b) results staged to shared memory, one bulk copy (shared -> global) per output and tile
  *_contig             (c) contiguous per-CTA tile ranges instead of the round-robin walk
  *_cta1, *_cta3       (d) 1 and 3 CTAs/SM
  ldg_1r1w / ldg_1r3w  the read side instead: no staging, each thread loads its elements with 8-byte loads (plain
                       stores); *_pertile: one CTA per tile instead of 2 CTAs/SM walking the tiles; *_res2: at
                       most 2 CTAs resident per SM; *_cta5: 5 CTAs/SM walking the tiles

Every launch is timed with CUDA events (--launches after --warmup); the whole table runs --rounds times in one
process.  Card name, power limit and SM clock are read in the same process.

    python benchmarks/hbm_mix.py [--n 1e9] [--launches 40] [--warmup 3] [--rounds 2]
"""
import argparse
import ctypes
import json
import os
import subprocess

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
LIB = os.path.join(ROOT, "ramba_b200", "lib", "librb200_probe.so")

# name -> (form, walk, CTAs/SM (0: one CTA per tile), outputs, ring depth, load form, resident cap (0: none))
ARMS = {
    "lib_1r3w_d2": (0, 0, 2, 3, 2, 0),
    "lib_1r3w_d6": (0, 0, 2, 3, 6, 0),
    "lib_1r1w": (0, 0, 2, 1, 2, 0),
    "shfl16": (1, 0, 2, 3, 2, 0),
    "bulk": (2, 0, 2, 3, 2, 0),
    "plain_contig": (0, 1, 2, 3, 2, 0),
    "shfl16_contig": (1, 1, 2, 3, 2, 0),
    "bulk_contig": (2, 1, 2, 3, 2, 0),
    "plain_cta1": (0, 0, 1, 3, 2, 0),
    "shfl16_cta1": (1, 0, 1, 3, 2, 0),
    "bulk_cta1": (2, 0, 1, 3, 2, 0),
    "plain_cta3": (0, 0, 3, 3, 2, 0),
    "shfl16_cta3": (1, 0, 3, 3, 2, 0),
    "bulk_cta3": (2, 0, 3, 3, 2, 0),
    "ldg_1r1w": (0, 0, 2, 1, 2, 1),
    "ldg_1r3w": (0, 0, 2, 3, 2, 1),
    "ldg_1r1w_pertile": (0, 0, 0, 1, 2, 1),
    "ldg_1r3w_pertile": (0, 0, 0, 3, 2, 1),
    "ldg_1r3w_pertile_res2": (0, 0, 0, 3, 2, 1, 2),
    "ldg_1r3w_cta5": (0, 0, 5, 3, 2, 1),
}


def card(dev):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader,nounits", "-i", str(dev)], capture_output=True, text=True)
    if out.returncode != 0:
        return {"card": None}
    name, plim, clk, clk_max = [x.strip() for x in out.stdout.strip().split(",")]
    return {"card": name, "power_limit_w": float(plim), "sm_clock_mhz": int(clk), "sm_clock_max_mhz": int(clk_max)}


def probe_lib(path=LIB):
    """The probe's shared object with the argument types of rb200_probe_run."""
    lib = ctypes.CDLL(path)
    lib.rb200_probe_run.restype = ctypes.c_int
    lib.rb200_probe_run.argtypes = [ctypes.c_int] * 7 + [ctypes.c_void_p] * 4 + [ctypes.c_longlong, ctypes.c_void_p]
    return lib


def timed(fn, launches, warmup):
    import torch

    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(launches)]
    for e0, e1 in ev:
        e0.record()
        fn()
        e1.record()
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e9)
    ap.add_argument("--launches", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--arms", default="copy,fill," + ",".join(ARMS))
    args = ap.parse_args()
    assert args.launches >= 30, "time at least 30 launches"
    import torch

    lib = probe_lib()
    n = int(args.n)
    dev = torch.cuda.current_device()
    a = torch.arange(n, dtype=torch.float64, device="cuda") / 1000.0
    outs = [torch.empty_like(a) for _ in range(3)]
    scale = (1.5, 2.5, 3.5)
    checked = set()
    for rnd in range(args.rounds):
        for arm in args.arms.split(","):
            res = {"arm": arm, "round": rnd, "n": n}
            if arm == "copy":
                ms = timed(lambda: outs[0].copy_(a), args.launches, args.warmup)
                rw = (1, 1)
            elif arm == "fill":
                ms = timed(lambda: outs[0].fill_(1.0), args.launches, args.warmup)
                rw = (0, 1)
            else:
                form, walk, minb, n_out, depth, load, resident = (ARMS[arm] + (0,))[:7]
                st = torch.cuda.current_stream().cuda_stream

                def run():
                    rc = lib.rb200_probe_run(form, walk, minb, load, resident, n_out, depth, a.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), n, st)
                    if rc != 0:
                        raise RuntimeError(rc)

                try:
                    run()
                except RuntimeError as e:
                    rc = e.args[0]
                    res["skipped"] = "fits %d CTAs/SM" % (-rc - 1) if -100 < rc < 0 else "error %d" % rc
                    print(json.dumps(res), flush=True)
                    continue
                if arm not in checked:
                    for j in range(n_out):
                        outs[j].fill_(0.0)
                    run()
                    for j in range(n_out):
                        assert torch.equal(outs[j], a * scale[j]), (arm, j)
                    checked.add(arm)
                ms = timed(run, args.launches, args.warmup)
                rw = (1, n_out)
                res.update({"form": ("plain", "shfl16", "bulk")[form], "walk": ("round_robin", "contiguous")[walk], "ctas_per_sm": minb or "one per tile",
                            "load": ("bulk_ring", "direct")[load], "ring_depth": depth if load == 0 else 0,
                            "resident_cap": resident or None})
            ms_mean = sum(ms) / len(ms)
            nbytes = 8 * n * (rw[0] + rw[1])
            res.update({"reads": rw[0], "writes": rw[1], "launches": len(ms), "kernel_ms": ms_mean, "kernel_ms_min": min(ms), "kernel_ms_max": max(ms),
                        "gbps": nbytes / ms_mean / 1e6})
            res.update(card(dev))
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
