"""Binning on one H100: histogram of 1e9 float64 and float32 into 256 and 4096 equal bins (data uniform over the range,
and every value in one bin), bincount of 1e9 int64 into 1000 and 10^6 bins (the global form), weighted bincount into 1000
bins and into 4096 bins (the slab form), and searchsorted of 1e9 float64 in 10^3 and 10^6 sorted values.

For each case: the kernel (rb200_histogram with its fold launches, or rb200_bin_search) by CUDA events, median of the
timed launches after warm-up; the traffic model over the kernel time and as a fraction of 3.35 TB/s (the H100 SXM
data-sheet HBM3 bandwidth).  The model counts the data once (element bytes), the weights once, 8 B per element of search
output and 8 B per bin of result.  The whole call is the public function to a synchronised result, wall clock, median of
10; torch.histc / torch.bincount / torch.searchsorted run on the same tensors in the same process.  The card's name and
power limit are read in the same process.  Prints one JSON line; writes nothing unless --out is given.

  python benchmarks/hist_bench.py [--reps 30] [--warmup 5] [--out FILE]"""
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
        raise SystemExit("hist_bench needs a CUDA device")
    import ramba_b200 as rb
    from ramba_b200 import _cabi, binning, blocks
    from ramba_b200.program import rb_dtype

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    gen = torch.Generator(device=dev).manual_seed(1)
    N = 10 ** 9
    results = []
    bad = torch.zeros(1, dtype=torch.int64, device=dev)

    def record(case, kernel_s, per_elem, B, view, weighted, table, wall_s, torch_s, torch_name):
        plan = _cabi.describe_hist_plan(view, weighted, table) if table is not None else "kernel=bin_search"
        nbytes = N * per_elem + B * 8
        results.append(dict(case, kernel_ms=kernel_s * 1e3, model_TBps=nbytes / kernel_s / 1e12, **{"share_of_3.35TBps": nbytes / HBM / kernel_s},
                            whole_call_ms=wall_s * 1e3, **{torch_name + "_ms": torch_s * 1e3}, plan=plan))
        print(json.dumps(results[-1]), file=sys.stderr)

    # ---- histogram: equal bins over [0, 1)
    for dt in (np.float64, np.float32):
        X = rb.empty((N,), dtype=dt)
        xt = blocks.block(X).interior()
        for skew in (False, True):
            if skew:
                xt.fill_(0.5)
            else:
                xt.uniform_(generator=gen)
            for B in (256, 4096):
                edges, uniform = binning._edges(X, B, (0.0, 1.0))
                dev_edges = binning._sorted_table(edges, edges.dtype)
                table = binning._table_for(X.dtype, edges, uniform, dev_edges, edges.dtype)
                view = blocks.index_view(X)
                out = torch.empty(B, dtype=torch.int64, device=dev)
                ks = _events(lambda: _cabi.histogram(view, rb_dtype(X.dtype), None, 0, table, out.data_ptr(), bad.data_ptr(), None, stream),
                             args.reps, args.warmup)
                h, _ = rb.histogram(X, bins=B, range=(0.0, 1.0))
                ref = torch.histc(xt, bins=B, min=0.0, max=1.0)
                exp = np.histogram(xt[: 1 << 20].cpu().numpy(), bins=B, range=(0.0, 1.0))[0]
                assert int(blocks.block(h).interior().sum()) == N and int(out.sum()) == N
                # torch.histc computes bins in its own arithmetic: compare totals with it, and NumPy on a prefix
                assert int(ref.sum()) == N
                hp, _ = rb.histogram(rb.fromarray(xt[: 1 << 20].cpu().numpy()), bins=B, range=(0.0, 1.0))
                assert np.array_equal(hp.asarray(), exp)
                wall = _wall(lambda: rb.histogram(X, bins=B, range=(0.0, 1.0)), 10, 2)
                ts = _events(lambda: torch.histc(xt, bins=B, min=0.0, max=1.0), max(5, args.reps // 3), 2)
                record({"call": "histogram", "dtype": np.dtype(dt).name, "bins": B, "one_bin": skew}, ks, np.dtype(dt).itemsize, B, view, False,
                       table, wall, ts, "torch_histc")
                del h, ref, hp, out
        del X, xt
        torch.cuda.empty_cache()
    # ---- bincount: counts (shared and global forms) and weights (shared and slab forms)
    X = rb.empty((N,), dtype=np.int64)
    xt = blocks.block(X).interior()
    Wt = rb.empty((N,), dtype=np.float64)
    wt = blocks.block(Wt).interior()
    wt.uniform_(generator=gen)
    for B, weighted in ((1000, False), (10 ** 6, False), (1000, True), (4096, True)):
        xt.random_(0, B, generator=gen)
        xt[-1] = B - 1
        table = _cabi.BinTable()
        table.form, table.n_bins = _cabi.BINS_INTEGER, B
        view = blocks.index_view(X)
        wview = blocks.index_view(Wt) if weighted else None
        out = torch.empty(B, dtype=torch.float64 if weighted else torch.int64, device=dev)
        nsc = _cabi.histogram_scratch_bytes(view, weighted, table)
        scr = torch.empty(max(nsc, 1), dtype=torch.uint8, device=dev)
        ks = _events(lambda: _cabi.histogram(view, _cabi.I64, wview, _cabi.F64 if weighted else 0, table, out.data_ptr(), bad.data_ptr(),
                                             scr.data_ptr() if nsc else None, stream), args.reps, args.warmup)
        call = (lambda: rb.bincount(X, weights=Wt)) if weighted else (lambda: rb.bincount(X))
        got = blocks.block(call()).interior()
        ref = torch.bincount(xt, weights=wt if weighted else None, minlength=B)
        if weighted:
            assert torch.allclose(got, ref, rtol=1e-9, atol=1e-6)
        else:
            assert torch.equal(got, ref)
        wall = _wall(call, 10, 2)
        ts = _events(lambda: torch.bincount(xt, weights=wt if weighted else None, minlength=B), max(5, args.reps // 3), 2)
        record({"call": "bincount", "dtype": "int64", "bins": B, "weighted": weighted}, ks, 8 + (8 if weighted else 0), B, view, weighted, table,
               wall, ts, "torch_bincount")
        del got, ref, out, scr
    del X, xt, Wt, wt
    torch.cuda.empty_cache()
    # ---- searchsorted of 1e9 float64 in sorted tables
    V = rb.empty((N,), dtype=np.float64)
    vt = blocks.block(V).interior()
    vt.uniform_(generator=gen)
    for m in (10 ** 3, 10 ** 6):
        a = np.sort(np.random.default_rng(m).random(m))
        at = torch.from_numpy(a).to(dev)
        out = torch.empty(N, dtype=torch.int64, device=dev)
        view = blocks.index_view(V)
        ks = _events(lambda: _cabi.bin_search(view, _cabi.F64, at.data_ptr(), m, _cabi.F64, _cabi.SEARCH_LEFT, out.data_ptr(), stream),
                     args.reps, args.warmup)
        assert torch.equal(out, torch.searchsorted(at, vt))
        wall = _wall(lambda: rb.searchsorted(a, V), 10, 2)
        ts = _events(lambda: torch.searchsorted(at, vt), max(5, args.reps // 3), 2)
        record({"call": "searchsorted", "dtype": "float64", "table": m}, ks, 16, 0, view, False, None, wall, ts, "torch_searchsorted")
        del out
        torch.cuda.empty_cache()
    line = json.dumps({"gpu": q, "results": results})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
