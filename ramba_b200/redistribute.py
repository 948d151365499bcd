"""reshape_copy: the C-order (linear) redistribution behind a general reshape (reference: ramba/ramba.py:9241-9277,
worker side RemoteState.reshape 2409-2499, which walks its block element by element in Python).

Both arrays are whole, block-partitioned arrays in C order.  A rank's block of either one is a set of RUNS - maximal
stretches of consecutive linear indices that are also consecutive in the rank's shard (whole rows of the trailing dims the
block covers completely).  The runs of a block all have the same length and form an arithmetic lattice, so they are generated
and intersected with NumPy index arithmetic, not per element:

    piece (s -> d) = run of rank s's SOURCE block  ∩  run of rank d's DESTINATION block.

Pieces with s == d are copied shard to shard; the others are packed into ONE buffer per peer, exchanged with one grouped
NCCL send / receive, and unpacked.  Consecutive pieces of equal length whose source and destination offsets advance by
constant steps are one 2-D strided copy - the library's op-list kernel with a MOV (`_pack_program`) over [pieces, length] -
so a reshape between regular partitions is a handful of launches per peer."""
import numpy as np


def block_runs(shape, start, size, contiguous_tail):
    """Runs of the block (start, size) of a C-order array of `shape`: (linear starts ascending, run length, index m of the dim a
    run walks; dims after m are covered completely).  `contiguous_tail` False (padded shard): runs never span rows."""
    k = len(shape)
    if k == 0 or any(int(n) <= 0 for n in size):
        return np.zeros(0, dtype=np.int64), 0, k - 1
    stride = [1] * k
    for j in range(k - 2, -1, -1):
        stride[j] = stride[j + 1] * int(shape[j + 1])
    m = k - 1
    if contiguous_tail:
        while m > 0 and int(size[m]) == int(shape[m]):
            m -= 1
    length = int(size[m]) * stride[m]
    starts = np.array([int(start[m]) * stride[m]], dtype=np.int64)
    for j in range(m - 1, -1, -1):
        starts = (np.arange(int(start[j]), int(start[j]) + int(size[j]), dtype=np.int64) * stride[j])[:, None] + starts[None, :]
        starts = starts.reshape(-1)
    return starts, length, m


def run_local_offsets(size, m, local_strides, origin):
    """Element offset in the shard of the first element of every run of a block (same order as block_runs)."""
    off = np.array([origin], dtype=np.int64)
    for j in range(m - 1, -1, -1):
        off = (np.arange(int(size[j]), dtype=np.int64) * int(local_strides[j]))[:, None] + off[None, :]
        off = off.reshape(-1)
    return off


def intersect_runs(a_start, a_len, b_start, b_len):
    """All non-empty intersections of two sorted families of equal-length, disjoint runs:
    (index into a, index into b, linear start, length), ordered by linear start.  a_len may also be one length per run
    of a (runs of a sorted and disjoint)."""
    a_len = np.broadcast_to(np.asarray(a_len, dtype=np.int64), np.shape(a_start))
    if len(a_start) == 0 or len(b_start) == 0 or not a_len.any() or b_len == 0:
        z = np.zeros(0, dtype=np.int64)
        return z, z, z, z
    lo = np.searchsorted(b_start + b_len, a_start, side="right")
    hi = np.searchsorted(b_start, a_start + a_len, side="left")
    cnt = np.maximum(hi - lo, 0)
    tot = int(cnt.sum())
    ia = np.repeat(np.arange(len(a_start), dtype=np.int64), cnt)
    first = np.repeat(np.cumsum(cnt) - cnt, cnt)
    ib = np.repeat(lo, cnt) + (np.arange(tot, dtype=np.int64) - first)
    s = np.maximum(a_start[ia], b_start[ib])
    e = np.minimum(a_start[ia] + a_len[ia], b_start[ib] + b_len)
    keep = e > s
    return ia[keep], ib[keep], s[keep], (e - s)[keep]


def strided_groups(length, src_off, dst_off):
    """Cut the piece list into maximal groups of consecutive pieces with one length and constant steps of both offsets:
    [(first piece, count, length, src step, dst step)] - each group is ONE 2-D strided copy."""
    n = len(length)
    out = []
    i = 0
    while i < n:
        j = i + 1
        ds = dd = 0
        if j < n and length[j] == length[i]:
            ds, dd = int(src_off[j] - src_off[i]), int(dst_off[j] - dst_off[i])
            j += 1
            while j < n and length[j] == length[i] and src_off[j] - src_off[j - 1] == ds and dst_off[j] - dst_off[j - 1] == dd:
                j += 1
        out.append((i, j - i, int(length[i]), ds, dd))
        i = j
    return out
