"""groupby programs: the 14 programs of the reference's ramba/tests/test_groupby.py, restated without xarray (the labels
are the day of year or the season of the same date ranges, computed with NumPy), plus cases the reference file does not
cover: every aggregate over int64 / int32 / float32 / float64 sources with empty groups, and a 3-D source grouped on its
middle axis.  Each program takes the module under test (the reference's `ramba` or `ramba_b200`) and returns
{name: NumPy array}.  tests/golden/make_groupby_golden.py runs them under the reference; test_groupby.py runs them here."""
import numpy as np


def doy(start, n):
    """Day of year - 1 of n consecutive days from `start` (pd.Timestamp(x).dayofyear - 1)."""
    d = np.datetime64(start) + np.arange(n)
    return (d - d.astype("datetime64[Y]").astype("datetime64[D]")).astype(np.int64)


def season(start, n):
    """(month % 12) // 3 of n consecutive days from `start`: 0 DJF, 1 MAM, 2 JJA, 3 SON."""
    d = np.datetime64(start) + np.arange(n)
    month = d.astype("datetime64[M]").astype(np.int64) % 12 + 1
    return (month % 12) // 3


def _np(x):
    return np.asarray(x.asarray() if hasattr(x, "asarray") else x)


def _anomaly(rb, x, labels, G, agg, keep_agg=True):
    gb = rb.fromarray(x).groupby(1, labels, num_groups=G)
    r = getattr(gb, agg)()
    out = {"final": _np(gb - r)}
    if keep_agg:
        out[agg] = _np(r)
    return out


# ---- the reference's test_groupby.py -----------------------------------------------------------------------------------
def mean_groupby1(rb):
    return _anomaly(rb, np.arange(1827).reshape(1, 1827), doy("2000-01-01", 1827), 366, "mean")


def mean_groupby2(rb):
    return _anomaly(rb, np.arange(2 * 1827).reshape(2, 1827), season("2000-01-01", 1827), 4, "mean")


def mean_groupby3(rb):
    x = np.random.default_rng(1234).random((2, 1827))
    return _anomaly(rb, x, doy("2000-01-01", 1827), 366, "mean")


def sum_groupby1(rb):
    return _anomaly(rb, np.arange(2 * 1827).reshape(2, 1827), doy("2000-01-01", 1827), 366, "sum")


def count_groupby1(rb):
    return _anomaly(rb, np.arange(2 * 1827).reshape(2, 1827), doy("2000-01-01", 1827), 366, "count")


def prod_groupby1(rb):
    return _anomaly(rb, np.arange(2 * 1827).reshape(2, 1827), doy("2000-01-01", 1827), 366, "prod")


def min_groupby1(rb):
    return _anomaly(rb, np.arange(1827).reshape(1, 1827), doy("2000-01-01", 1827), 366, "min")


def max_groupby1(rb):
    return _anomaly(rb, np.arange(2 * 1827).reshape(2, 1827), doy("2000-01-01", 1827), 366, "max")


def var_groupby1(rb):
    gb = rb.fromarray(np.arange(1827).reshape(1, 1827)).groupby(1, doy("2000-01-01", 1827), num_groups=366)
    return {"var": _np(gb.var())}


def std_groupby1(rb):
    gb = rb.fromarray(np.arange(1827).reshape(1, 1827)).groupby(1, doy("2000-01-01", 1827), num_groups=366)
    return {"std": _np(gb.std())}


def _mean_view(rb, total, view):
    a = view(rb.fromarray(np.arange(total[0] * total[1]).reshape(total)))
    gb = a.groupby(1, doy("2001-01-01", a.shape[1]), num_groups=365)
    m = gb.mean()
    return {"mean": _np(m), "final": _np(gb - m)}


def mean_groupby_slice1(rb):
    return _mean_view(rb, (1, 400), lambda a: a[:, 25:25 + 365])


def mean_groupby_transpose1(rb):
    return _mean_view(rb, (365, 1), lambda a: a.T)


def mean_groupby_slice_transpose1(rb):
    return _mean_view(rb, (400, 1), lambda a: a.T[:, 25:25 + 365])


def mean_groupby_slice_transpose2(rb):
    return _mean_view(rb, (400, 1), lambda a: a[25:25 + 365, :].T)


REFERENCE_PROGRAMS = [mean_groupby1, mean_groupby2, mean_groupby3, sum_groupby1, count_groupby1, prod_groupby1, min_groupby1,
                      max_groupby1, var_groupby1, std_groupby1, mean_groupby_slice1, mean_groupby_transpose1,
                      mean_groupby_slice_transpose1, mean_groupby_slice_transpose2]

# ---- every aggregate, every kernel dtype, empty groups, a middle axis -------------------------------------------------
AGGS = ("sum", "prod", "min", "max", "count", "mean", "var", "std")


def _every_aggregate(rb, x, dim, labels, G):
    gb = rb.fromarray(x).groupby(dim, labels, num_groups=G)
    out = {agg: _np(getattr(gb, agg)()) for agg in AGGS}
    out["final"] = _np(gb - gb.mean())
    return out


def _small(shape, dtype, seed):
    return np.random.default_rng(seed).integers(1, 4, size=shape).astype(dtype)  # 1..3: products stay exact


def _labels_with_empty_groups(n, seed):
    lab = np.random.default_rng(seed).integers(0, 6, size=n)
    lab[lab == 2] = 0  # groups 2, 6 and 7 of G = 8 stay empty
    return lab


def every_aggregate_int64(rb):
    return _every_aggregate(rb, _small((3, 24), np.int64, 1), 1, _labels_with_empty_groups(24, 2), 8)


def every_aggregate_int32(rb):
    return _every_aggregate(rb, _small((3, 24), np.int32, 3), 1, _labels_with_empty_groups(24, 4), 8)


def every_aggregate_float32(rb):
    return _every_aggregate(rb, _small((3, 24), np.float32, 5) * np.float32(0.5), 1, _labels_with_empty_groups(24, 6), 8)


def every_aggregate_float64(rb):
    return _every_aggregate(rb, _small((3, 24), np.float64, 7) * 0.25, 1, _labels_with_empty_groups(24, 8), 8)


def middle_axis_3d(rb):
    return _every_aggregate(rb, _small((4, 30, 5), np.float64, 9), 1, _labels_with_empty_groups(30, 10), 8)


def first_axis_season(rb):
    x = np.random.default_rng(11).random((1827, 3))
    return _every_aggregate(rb, x, 0, season("2000-01-01", 1827), 4)


EXTRA_PROGRAMS = [every_aggregate_int64, every_aggregate_int32, every_aggregate_float32, every_aggregate_float64, middle_axis_3d,
                  first_axis_season]
PROGRAMS = REFERENCE_PROGRAMS + EXTRA_PROGRAMS
