"""Integer-array indexing programs written against a NumPy-like module `app`: the reference's own
TestBasic::test_fancy_indexing1-4 (ramba/tests/test_distributed_array.py:874-917) and further cases the reference can run.
tests/golden/make_fancy_golden.py runs them under the reference (`import ramba`) and stores the outputs in
fancy_golden.npz; tests/test_fancy_indexing.py runs them under ramba_b200 (and NumPy) and compares.  Each program returns a
dict of NumPy arrays."""
import numpy as onp


def fancy_indexing1(app):
    a = app.ones((11, 21, 31, 41), dtype=int)
    b = a[7, 5, [2, 6, 1], 3:6]
    c = a[None, [[3, 4, 7]], 4, [[3], [2], [7], [1]]]
    d = a[None, [[2, 3, 1]], 4, None, [[1], [7]], 4:9]
    return {"shapes": onp.array([list(b.shape) + [0] * 3, list(c.shape) + [0], list(d.shape)])}


def fancy_indexing2(app):
    a = app.arange(500)
    b = a[::7]
    c = app.fromfunction(lambda i, j: (i + j) % 70, (50, 20), dtype=int)
    return {"d": onp.asarray(b[c])}


def fancy_indexing3(app):
    a = app.arange(500)
    b = a[::2]
    c = app.fromfunction(lambda i, j: i + j * 100, (50, 3), dtype=int)
    b[c] = 1
    return {"a": onp.asarray(a)}


def fancy_indexing4(app):
    a = app.arange(500)
    b = a[::2]
    c = app.fromfunction(lambda i, j: i + j * 100, (50, 3), dtype=int)
    d = app.fromfunction(lambda i, j: (i - j), (50, 100), dtype=int)
    b[c] = d[:, 48:51]
    return {"a": onp.asarray(a)}


def gather_2d_lists(app):
    a = app.fromfunction(lambda i, j: i * 100 + j, (30, 40), dtype=int)
    return {"rows": onp.asarray(a[[3, 29, 0, 7]]), "pairs": onp.asarray(a[[1, 2, 28], [39, 0, 5]]),
            "cols": onp.asarray(a[5:25:4, [6, 1, 33]])}


def gather_negative(app):
    a = app.fromfunction(lambda i: i * 3, (100,), dtype=int)
    return {"neg": onp.asarray(a[[-1, -100, 50, -7]])}


def gather_by_array(app):
    a = app.fromfunction(lambda i, j: i - 2 * j, (60, 25), dtype=int)
    c = app.fromfunction(lambda i, j: (i * 7 + j * 3) % 60, (12, 5), dtype=int)
    return {"g": onp.asarray(a[c])}


def scatter_array_value(app):
    a = app.zeros((50, 8), dtype=int)
    a[[4, 17, 49], 2:6] = app.fromfunction(lambda i, j: i * 10 + j + 1, (3, 4), dtype=int)
    return {"a": onp.asarray(a)}


PROGRAMS = [fancy_indexing1, fancy_indexing2, fancy_indexing3, fancy_indexing4, gather_2d_lists, gather_negative,
            gather_by_array, scatter_array_value]
