"""rb200_arg_reduce on one H100: argmax of 1e9 float64 and 1e9 float32 over every axis (global form), of a
(65536, 4096) float64 array along axis 1 (row form) and axis 0 (column form), and nanargmax of the 1e9 float64 case.

For each case: kernel time (CUDA events around one rb200_arg_reduce, median of the timed launches after warm-up),
source bytes over that time and over 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth; the roof of a one-read
reduction), whole-call wall time of the public API to a host result, and torch.argmax on the same tensor in the same
process as a comparator.  The card's name and power limit are read in the same process.  Prints one JSON line; writes
nothing unless --out is given.

  python benchmarks/argreduce_bench.py [--reps 30] [--warmup 5] [--out FILE]"""
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
        r = fn()
        if hasattr(r, "asarray"):
            r.asarray()
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
        raise SystemExit("argreduce_bench needs a CUDA device")
    import ramba_b200 as rb
    from ramba_b200 import _cabi, blocks

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(1)
    cases = [("argmax_f64_1e9", (10 ** 9,), torch.float64, None, _cabi.ARG_MAX),
             ("argmax_f32_1e9", (10 ** 9,), torch.float32, None, _cabi.ARG_MAX),
             ("nanargmax_f64_1e9", (10 ** 9,), torch.float64, None, _cabi.ARG_NANMAX),
             ("argmax_f64_65536x4096_axis1", (65536, 4096), torch.float64, 1, _cabi.ARG_MAX),
             ("argmax_f64_65536x4096_axis0", (65536, 4096), torch.float64, 0, _cabi.ARG_MAX)]
    results = []
    for name, shape, tdt, axis, op in cases:
        npdt = np.float64 if tdt == torch.float64 else np.float32
        A = rb.empty(shape, dtype=npdt)
        sh = blocks.block(A)
        t = sh.interior()
        t.uniform_(generator=gen)
        t.view(-1)[len(t.view(-1)) * 3 // 4] = 2.0  # a known maximum
        view = blocks.index_view(A)
        cax = _cabi.ARG_ALL_AXES if axis is None else axis
        n_out = 1 if axis is None else shape[1 - axis]
        idx = torch.empty(n_out, dtype=torch.int64, device=dev)
        key = torch.empty(n_out, dtype=torch.int64, device=dev)
        nbytes = _cabi.arg_reduce_scratch_bytes(view, cax)
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        o, g = _cabi.arg_coords([0] * len(shape), [shape[1], 1] if len(shape) == 2 else [1])
        stream = torch.cuda.current_stream(dev).cuda_stream

        def kernel():
            _cabi.arg_reduce(view, _cabi.F64 if npdt == np.float64 else _cabi.F32, cax, op, o, g, idx.data_ptr(), key.data_ptr(), scratch.data_ptr(),
                             stream)

        k_s = _events(kernel, args.reps, args.warmup)
        fn = {_cabi.ARG_MAX: rb.argmax, _cabi.ARG_NANMAX: rb.nanargmax}[op]
        wall_s = _wall(lambda: fn(A, axis=axis), max(5, args.reps // 3), 2)
        ref = torch.argmax(t) if axis is None else torch.argmax(t, dim=axis)
        got = fn(A, axis=axis)
        got = np.asarray(got.asarray() if hasattr(got, "asarray") else got)
        assert np.array_equal(got, ref.cpu().numpy()), name
        torch_s = _events(lambda: torch.argmax(t) if axis is None else torch.argmax(t, dim=axis), args.reps, args.warmup)
        src_bytes = int(np.prod(shape)) * t.element_size()
        results.append({"case": name, "form": _cabi.group_plan_fields(_cabi.describe_arg_plan(view, cax))["form"], "kernel_ms": k_s * 1e3,
                        "kernel_TBps": src_bytes / k_s / 1e12, "share_of_3.35TBps": src_bytes / HBM / k_s, "wall_ms": wall_s * 1e3,
                        "torch_argmax_ms": torch_s * 1e3})
        del A, sh, t, scratch
        torch.cuda.empty_cache()
    line = json.dumps({"gpu": q, "results": results})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
