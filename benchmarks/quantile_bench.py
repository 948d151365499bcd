"""Order statistics on one H100: the global median of 1e9 float64 (uniform, normal and all-equal data) and of 1e9
float32, percentile(a, [1, 25, 50, 75, 99]) and nanmedian with 10 % NaN of 1e9 float64, and median(axis=1) / median(axis=0)
of a (65536, 4096) float64 array.

For each case: the kernel time, the sum over the call's select launches (each count pass with its memsets, each choose,
or the one row launch) of CUDA events recorded around that launch, median over the timed repetitions after warm-up, also
per count pass; the passes, which of them read the data and which the compacted candidates; the model bytes (the data
once per launch that reads it, 8 B per candidate key written or read) over the kernel time and as a fraction of 3.35
TB/s (the H100 SXM data-sheet HBM3 bandwidth).  The whole call is the public function to a synchronised result, wall
clock, median of 10 (host reads between passes and NumPy's finish included).  torch.median, torch.kthvalue and torch.quantile
(where its input-size limit allows) run on the same tensors in the same process.  The card's name and power limit are
read in the same process.  Prints one JSON line; writes nothing unless --out is given.

  python benchmarks/quantile_bench.py [--reps 30] [--warmup 3] [--n 1000000000] [--out FILE]"""
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


class _Trace:
    """While active: CUDA events around every select launch of the backend, the mode of each count pass and the
    candidate keys it wrote or read; the backend's own methods are restored on exit."""

    NAMES = ("select_count", "select_choose", "select_rows")

    def __init__(self, RT):
        self.be = RT.be()

    def __enter__(self):
        self.modes, self.cand, self.rows, self.events = [], 0, 0, []
        for name in self.NAMES:
            setattr(self.be, name, self._timed(name, getattr(type(self.be), name).__get__(self.be)))
        return self

    def __exit__(self, *exc):
        for name in self.NAMES:
            delattr(self.be, name)
        return False

    def _timed(self, name, fn):
        def call(*a):
            if name == "select_count":
                st, mode = a[3], a[5]
                self.modes.append(mode)
                self.cand += 8 * int(st.cand_cap) if mode != 0 else 0
            self.rows += name == "select_rows"
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*a)
            e1.record()
            self.events.append((e0, e1))
            return out

        return call

    def kernel_s(self):
        torch.cuda.synchronize()
        return sum(e0.elapsed_time(e1) for e0, e1 in self.events) * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--n", type=int, default=10 ** 9)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("quantile_bench needs a CUDA device")
    import ramba_b200 as rb
    from ramba_b200 import _cabi
    from ramba_b200.runtime import RT

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    n = args.n
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    results = []

    def case(name, call, data_t, torch_calls):
        tr = _Trace(RT)
        for _ in range(args.warmup):
            call()
        times = []
        for _ in range(args.reps):
            with tr:
                call()
                times.append(tr.kernel_s())
        kt = float(np.median(times))
        modes, rows = list(tr.modes), tr.rows
        full = sum(1 for m in modes if m != _cabi.SELECT_CAND) + rows
        model = full * data_t.numel() * data_t.element_size() + tr.cand
        wall = _wall(call, 10, 1)
        tt = {}
        for tn, tf in torch_calls:
            try:
                tt[tn] = _events(tf, 10, 2)
            except RuntimeError as ex:  # (torch.quantile's input-size limit)
                tt[tn] = "not run: %s" % str(ex).split("\n")[0][:80]
        results.append({"case": name, "passes": len(modes) or None, "row_launches": rows, "count_modes": modes, "full_reads": full,
                        "model_bytes": model, "kernel_s": kt, "kernel_s_per_count_pass": kt / len(modes) if modes else None,
                        "GBps": model / kt / 1e9, "of_hbm": model / kt / HBM, "whole_call_s": wall, "torch_s": tt})
        print(json.dumps(results[-1]), file=sys.stderr)

    for dt, dname in ((torch.float64, "float64"), (torch.float32, "float32")):
        for kind in ("uniform", "normal", "equal"):
            if dt == torch.float32 and kind != "normal":
                continue
            if kind == "uniform":
                t = torch.rand(n, dtype=dt, device=dev, generator=g)
            elif kind == "normal":
                t = torch.randn(n, dtype=dt, device=dev, generator=g)
            else:
                t = torch.full((n,), 0.5, dtype=dt, device=dev)
            X = rb.fromarray(t.cpu().numpy())
            xk = X
            case("median %s %s n=%d" % (dname, kind, n), lambda: rb.median(xk), t,
                 [("torch.median", lambda: torch.median(t)), ("torch.kthvalue", lambda: torch.kthvalue(t, (n + 1) // 2)),
                                   ("torch.quantile", lambda: torch.quantile(t, 0.5))])
            if dt == torch.float64 and kind == "normal":
                qq = torch.tensor([0.01, 0.25, 0.5, 0.75, 0.99], dtype=dt, device=dev)
                case("percentile [1,25,50,75,99] float64 normal", lambda: rb.percentile(xk, [1, 25, 50, 75, 99]), t,
                     [("torch.quantile", lambda: torch.quantile(t, qq))])
                tn = t.clone()
                tn[torch.rand(n, device=dev, generator=g) < 0.1] = float("nan")
                XN = rb.fromarray(tn.cpu().numpy())
                case("nanmedian float64 normal 10% NaN", lambda: rb.nanmedian(XN), tn,
                     [("torch.nanmedian", lambda: torch.nanmedian(tn))])
                del tn, XN
            del X, xk, t
            torch.cuda.empty_cache()
    t = torch.randn((65536, 4096), dtype=torch.float64, device=dev, generator=g)
    Y = rb.fromarray(t.cpu().numpy())
    case("median axis=1 (65536, 4096) float64", lambda: rb.median(Y, axis=1), t,
         [("torch.median dim=1", lambda: torch.median(t, dim=1)), ("torch.kthvalue dim=1", lambda: torch.kthvalue(t, 2048, dim=1))])
    # the row kernel alone (rb200_select_rows on the same view, ranks 2047 and 2048)
    from ramba_b200 import blocks

    view = blocks.index_view(Y)
    table = torch.tensor([2047, 2048], dtype=torch.int64, device=dev)
    keys, nans = torch.empty(65536 * 2, dtype=torch.int64, device=dev), torch.empty(65536, dtype=torch.int64, device=dev)
    kt = _events(lambda: _cabi.select_rows(view, _cabi.F64, 4096, 2, table.data_ptr(), False, keys.data_ptr(), nans.data_ptr()),
                 args.reps, args.warmup)
    results.append({"case": "rb200_select_rows alone, (65536, 4096) float64", "kernel_s": kt, "of_hbm": t.numel() * 8 / kt / HBM})
    print(json.dumps(results[-1]), file=sys.stderr)
    case("median axis=0 (65536, 4096) float64", lambda: rb.median(Y, axis=0), t,
         [("torch.median dim=0", lambda: torch.median(t, dim=0)), ("torch.kthvalue dim=0", lambda: torch.kthvalue(t, 32768, dim=0))])
    line = json.dumps({"gpu": q, "results": results})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
