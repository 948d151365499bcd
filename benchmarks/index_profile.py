"""torch.profiler breakdown of one `a[idx]` call on one GPU: which kernels the address-stream flush (lin and its
out-of-range count) and the gather launch, and how long each takes.  Writes nothing; prints the table.

    python benchmarks/index_profile.py [--n 1e9]"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    import ramba_b200 as rb

    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e9)
    n = int(ap.parse_args().n)
    A = rb.random.random(n)
    idx = rb.arange(n)
    A.instantiate()
    idx.instantiate()
    rb.sync()
    for _ in range(2):
        A[idx]
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        r = A[idx]
        torch.cuda.synchronize()
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=15))
    del r


if __name__ == "__main__":
    main()
