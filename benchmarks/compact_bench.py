"""Stream compaction on one H100: extract(mask, x) of 1e9 float64 with a bool mask and flatnonzero of 1e9 bool, at
densities 0, 0.01, 0.5 and 1, and nonzero of a (32768, 32768) float32 at density 0.5.

For each case: each pass (rb200_compact_count, the rb200_cumulative scan of the chunk counts, rb200_compact) by CUDA
events, median of the timed launches after warm-up; the traffic model over the summed kernel time and as a fraction of
3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth).  The model counts the condition twice (count and compact pass), the
whole value stream of `extract` once (8 B per element: at density 1/2 every sector is touched), and the written
payload: per element 2c + 8 + 8p for extract, 2c + 8p for flatnonzero and 2c + 16p for the 2-d nonzero (c: condition
bytes, p: density).  The whole call is the public function to a synchronised result, wall clock, median of 10;
torch.masked_select / torch.nonzero run on the same tensors in the same process.  The card's name and power limit are
read in the same process.  Prints one JSON line; writes nothing unless --out is given.

  python benchmarks/compact_bench.py [--reps 30] [--warmup 5] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM = 3.35e12


def _events(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    return float(np.median(ts))


def _wall(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("compact_bench needs a CUDA device")
    import ramba_b200 as rb
    from ramba_b200 import _cabi, blocks
    from ramba_b200.program import rb_dtype

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    gen = torch.Generator(device=dev).manual_seed(1)
    N = 10 ** 9
    X = rb.empty((N,), dtype=np.float64)
    xt = blocks.block(X).interior()
    xt.uniform_(generator=gen)
    cases = [("extract", d, (N,), np.bool_) for d in (0.0, 0.01, 0.5, 1.0)] + [("flatnonzero", d, (N,), np.bool_) for d in (0.0, 0.01, 0.5, 1.0)] + \
        [("nonzero", 0.5, (32768, 32768), np.float32)]
    results = []
    for fn, density, shape, cdt in cases:
        M = rb.empty(shape, dtype=cdt)
        mt = blocks.block(M).interior()
        u = torch.rand(shape, generator=gen, device=dev, dtype=torch.float32)
        if cdt == np.bool_:
            mt.copy_((u < density).to(torch.uint8))
        else:
            mt.copy_(torch.where(u < density, u + 1.0, torch.zeros_like(u)))
        del u
        n = int(np.prod(shape))
        cond = blocks.index_view(M)
        code = rb_dtype(M.dtype)
        cpr = -(-n // _cabi.COMPACT_CHUNK)
        counts = torch.empty(cpr, dtype=torch.int64, device=dev)
        incl = torch.empty(cpr, dtype=torch.int64, device=dev)
        scr = torch.empty(_cabi.cumulative_scratch_bytes(1, cpr, 1), dtype=torch.uint8, device=dev)
        base = torch.zeros(1, dtype=torch.int64, device=dev)
        sel = int(mt.count_nonzero())
        form = {"extract": _cabi.COMPACT_VALUES, "flatnonzero": _cabi.COMPACT_FLAT, "nonzero": _cabi.COMPACT_COORDS}[fn]
        k = len(shape) if fn == "nonzero" else 1
        outs = [torch.empty(max(sel, 1), dtype=torch.float64 if fn == "extract" else torch.int64, device=dev) for _ in range(k)]
        vview = blocks.index_view(X) if fn == "extract" else None
        gst = [shape[1], 1] if len(shape) == 2 else [1]
        count_s = _events(lambda: _cabi.compact_count(cond, code, n, counts.data_ptr(), stream), args.reps, args.warmup)
        scan_s = _events(lambda: _cabi.cumulative(counts.data_ptr(), incl.data_ptr(), _cabi.I64, 1, cpr, 1, _cabi.RED_ADD, None, None, scr.data_ptr(),
                                                  stream), args.reps, args.warmup)
        compact_s = _events(lambda: _cabi.compact(cond, code, n, counts.data_ptr(), incl.data_ptr(), base.data_ptr(), form, vview, [0] * len(shape), gst,
                                                  [o.data_ptr() for o in outs], stream), args.reps, args.warmup)
        call = {"extract": lambda: rb.extract(M, X), "flatnonzero": lambda: rb.flatnonzero(M), "nonzero": lambda: rb.nonzero(M)}[fn]
        wall_s = _wall(call, 10, 2)
        # the engine's result against torch's on the same tensors
        if fn == "extract":
            ref = torch.masked_select(xt, mt.bool())
            torch_fn = lambda: torch.masked_select(xt, mt.bool())  # noqa: E731
            got = [blocks.block(call()).interior()]
            refs = [ref]
        else:
            ref = torch.nonzero(mt.reshape(-1) if fn == "flatnonzero" else mt)
            torch_fn = (lambda: torch.nonzero(mt.reshape(-1))) if fn == "flatnonzero" else (lambda: torch.nonzero(mt))  # noqa: E731
            got = [blocks.block(a).interior() for a in (call() if fn == "nonzero" else (call(),))]
            refs = [ref[:, d] for d in range(ref.shape[1])]
        assert all(torch.equal(g, r) for g, r in zip(got, refs)), (fn, density)
        del got, refs, ref
        torch_s = _events(torch_fn, max(5, args.reps // 3), 2)
        c = M.dtype.itemsize
        per = 2 * c + (8 + 8 * density if fn == "extract" else 8 * density if fn == "flatnonzero" else 16 * density)
        ksum = count_s + scan_s + compact_s
        results.append({"call": fn, "density": density, "shape": list(shape), "cond": str(M.dtype), "selected": sel,
                        "count_ms": count_s * 1e3, "scan_ms": scan_s * 1e3, "compact_ms": compact_s * 1e3, "kernels_ms": ksum * 1e3,
                        "model_TBps": n * per / ksum / 1e12, "share_of_3.35TBps": n * per / HBM / ksum, "whole_call_ms": wall_s * 1e3,
                        ("torch_masked_select_ms" if fn == "extract" else "torch_nonzero_ms"): torch_s * 1e3,
                        "plan": _cabi.describe_compact_plan(cond, n)})
        print(json.dumps(results[-1]), file=sys.stderr)
        del M, mt, outs, counts, incl, scr
        torch.cuda.empty_cache()
    line = json.dumps({"gpu": q, "results": results})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
