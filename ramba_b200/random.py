"""`ramba_b200.random`: random arrays drawn on the GPU, with values that do not depend on the number of ranks.

The reference fills each worker's block with NumPy's generator seeded by `seed + worker_num` (ramba/ramba.py:3824-3825),
so its arrays change with the worker count.  Here element i of a draw is a pure function of (seed, draw number, i):
Philox4x32-10 keyed by `splitmix64(splitmix64(seed) ^ draw_number)` and counted by the global C-order index i
(RB200_OP_PHILOX, include/ramba_b200.h).  So

  * the same seed gives the same arrays on any number of GPUs and under any partition;
  * a draw is an ordinary deferred statement (like `arange`): `x = rand(N); y = rand(N); ((x*x + y*y) < 1).sum()` runs
    as one fused kernel that reads nothing from memory;
  * the draw number is taken when the function is called, so DAG order, pruning, fusion and RAMBA_NO_DAG=1 cannot
    change the values, and a draw whose result is never used still advances the counter.

The streams are not NumPy's: the same seed gives different numbers than `numpy.random` (NumPy's generators are
sequential and cannot be evaluated per element in parallel).  `size=None` returns a host scalar from a NumPy generator
seeded with the same seed, as the reference does.
"""
import numbers
import os

import numpy as np
import torch

from . import _cabi as cabi
from . import common
from . import ramba as _r
from .program import E, Iota
from .runtime import RT

_M64 = (1 << 64) - 1


def splitmix64(x):
    """One step of the splitmix64 output function (Steele, Lea, Flood, OOPSLA'14) on a 64-bit integer."""
    z = (x + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def draw_key(seed, draw_number):
    """The 64-bit Philox key of draw `draw_number` of a generator seeded with `seed`."""
    return splitmix64(splitmix64(seed) ^ (draw_number & _M64))


def _check_seed(seed):
    if isinstance(seed, (bool, np.bool_)) or not isinstance(seed, numbers.Integral):
        raise ValueError("seed must be a non-negative integer below 2**64, not %r" % (seed,))
    seed = int(seed)
    if seed < 0 or seed > _M64:
        raise ValueError("seed must be a non-negative integer below 2**64, not %d" % seed)
    return seed


def _fresh_seed():
    """A seed from os.urandom on rank 0, broadcast so that every SPMD rank draws the same arrays."""
    seed = int.from_bytes(os.urandom(8), "little")
    if common.num_workers > 1:
        t = torch.tensor([seed - (1 << 64) if seed >= (1 << 63) else seed], dtype=torch.int64).to(RT.device)
        RT.broadcast(t, 0)
        seed = int(t.cpu().item()) & _M64
    return seed


def _shape(size):
    if isinstance(size, numbers.Integral):
        size = (size,)
    shape = tuple(int(s) for s in size)
    if any(s < 0 for s in shape):
        raise ValueError("negative dimensions are not allowed")
    return shape


def _linear_index(shape):
    """The global C-order linear index of the element as an index expression (Horner form over the IOTAs)."""
    idx = Iota(0)
    for d in range(1, len(shape)):
        idx = E("add", E("mul", idx, shape[d]), Iota(d))
    return idx


class _State:
    """A seed and the number of draws made since it was set."""

    def __init__(self, seed=None):
        self._seed = None if seed is None else _check_seed(seed)
        self._draws = 0
        self._host = None

    def reseed(self, seed):
        self.__init__(seed)

    def _key(self):
        if self._seed is None:
            self._seed = _fresh_seed()
        k = draw_key(self._seed, self._draws)
        self._draws += 1
        return k - (1 << 64) if k >= (1 << 63) else k  # (the int64 scalar with the key's bits)

    def host(self):
        """NumPy generator for scalar draws (size=None), seeded with the same seed."""
        if self._host is None:
            if self._seed is None:
                self._seed = _fresh_seed()
            self._host = np.random.default_rng(self._seed)
        return self._host

    def draw(self, size, form, dtype, tail=None, bound=None):
        """A deferred array of shape `size` holding draw `form` (PHILOX_*) followed by `tail(expr)`."""
        shape = _shape(size)
        if shape == ():
            raise ValueError("size=() is not supported: pass size=None for a scalar")
        key = self._key()  # taken now, whether or not the array is ever computed
        res = _r.empty(shape, dtype=dtype)
        if 0 in shape:
            return res
        args = (_linear_index(shape), key) + (() if bound is None else (bound,))
        expr = E("philox", *args, imm=form)
        if tail is not None:
            expr = tail(expr)
        _r.DAG.assign(res, expr)
        return res

    # ---- the distributions
    def random(self, size=None, dtype=np.float64):
        dtype = np.dtype(dtype)
        if dtype not in (np.dtype(np.float64), np.dtype(np.float32)):
            raise ValueError("random: dtype must be float64 or float32, not %s" % dtype)
        if size is None:
            return self.host().random(dtype=dtype)
        form = cabi.PHILOX_UNIFORM32 if dtype == np.float32 else cabi.PHILOX_UNIFORM64
        return self.draw(size, form, dtype)

    def uniform(self, low=0.0, high=1.0, size=None):
        low, high = float(low), float(high)
        if not low < high:
            raise ValueError("uniform: low must be below high (got %r, %r)" % (low, high))
        if size is None:
            return self.host().uniform(low, high)
        span = high - low
        return self.draw(size, cabi.PHILOX_UNIFORM64, np.float64, tail=lambda u: E("add", low, E("mul", span, u)))

    def standard_normal(self, size=None):
        if size is None:
            return self.host().standard_normal()
        return self.draw(size, cabi.PHILOX_NORMAL64, np.float64)

    def normal(self, loc=0.0, scale=1.0, size=None):
        loc, scale = float(loc), float(scale)
        if scale < 0:
            raise ValueError("normal: scale must be non-negative")
        if size is None:
            return self.host().normal(loc, scale)
        return self.draw(size, cabi.PHILOX_NORMAL64, np.float64, tail=lambda z: E("add", loc, E("mul", scale, z)))

    def integers(self, low, high=None, size=None, dtype=np.int64):
        if high is None:
            low, high = 0, low
        low, high = int(low), int(high)
        if not low < high:
            raise ValueError("randint: low must be below high (got %d, %d)" % (low, high))
        n = high - low
        if n >= (1 << 63) or low < -(1 << 63) or high > (1 << 63):
            raise ValueError("randint: the range must hold fewer than 2**63 values and fit in int64")
        if size is None:
            return self.host().integers(low, high, dtype=dtype)
        tail = None if low == 0 else (lambda x: E("add", x, low))
        res = self.draw(size, cabi.PHILOX_INTEGER, np.int64, tail=tail, bound=n)
        return res if np.dtype(dtype) == np.int64 else res.astype(dtype)

    def choice(self, a, size=None, replace=True, p=None):
        """`a[integers(0, len(a), size)]` (a range when `a` is an int): one draw, the same bits at any rank count."""
        if not replace:
            raise NotImplementedError("choice(replace=False) is not supported (it needs a permutation)")
        if p is not None:
            raise NotImplementedError("choice(p=...) is not supported")
        if isinstance(a, numbers.Integral):
            return self.integers(0, int(a), size)
        pool = a if isinstance(a, _r.ndarray) else np.asarray(a)
        if pool.ndim != 1:
            raise ValueError("choice: a must be an int or a 1-D array")
        if len(pool) == 0:
            raise ValueError("choice: a cannot be empty")
        idx = self.integers(0, len(pool), size)
        if size is None:
            return pool[int(idx)]
        return pool[idx] if isinstance(pool, _r.ndarray) else _r.fromarray(pool)[idx]


_global = _State()


# ---- the module-level (legacy NumPy) interface
def seed(x=None):
    """Re-seed the module-level generator; None takes a fresh seed from os.urandom (shared by all ranks)."""
    _global.reseed(x)


def random(size=None, dtype=np.float64):
    """Uniform float64 (or float32) values in [0, 1)."""
    return _global.random(size, dtype)


random_sample = random


def rand(*shape):
    return _global.random(shape if shape else None)


def randn(*shape):
    return _global.standard_normal(shape if shape else None)


def uniform(low=0.0, high=1.0, size=None):
    return _global.uniform(low, high, size)


def normal(loc=0.0, scale=1.0, size=None):
    return _global.normal(loc, scale, size)


def standard_normal(size=None):
    return _global.standard_normal(size)


def randint(low, high=None, size=None, dtype=np.int64):
    """Integers in [low, high) (or [0, low) when high is None)."""
    return _global.integers(low, high, size, dtype)


def choice(a, size=None, replace=True, p=None):
    """Elements of the 1-D array `a` (or of range(a)) picked uniformly with replacement; see _State.choice."""
    return _global.choice(a, size, replace, p)


class Generator:
    """`numpy.random.Generator` subset: random, normal, standard_normal, uniform, integers, choice."""

    def __init__(self, seed=None):
        self._state = _State(seed)

    def random(self, size=None, dtype=np.float64, out=None):
        if out is not None:
            raise NotImplementedError("Generator.random: out= is not supported")
        return self._state.random(size, dtype)

    def normal(self, loc=0.0, scale=1.0, size=None):
        return self._state.normal(loc, scale, size)

    def standard_normal(self, size=None):
        return self._state.standard_normal(size)

    def uniform(self, low=0.0, high=1.0, size=None):
        return self._state.uniform(low, high, size)

    def integers(self, low, high=None, size=None, dtype=np.int64, endpoint=False):
        if endpoint:
            if high is None:
                low, high = 0, low
            high = int(high) + 1
        return self._state.integers(low, high, size, dtype)

    def choice(self, a, size=None, replace=True, p=None):
        return self._state.choice(a, size, replace, p)


def default_rng(seed=None):
    return Generator(seed)


class RandomState:
    """`numpy.random.RandomState` subset: random, random_sample, rand, randn, uniform, normal, standard_normal,
    randint, choice.  Any other method raises NotImplementedError."""

    _METHODS = ("random", "random_sample", "rand", "randn", "uniform", "normal", "standard_normal", "randint", "choice", "seed")

    def __init__(self, seed=None):
        self._state = _State(seed)

    def seed(self, seed=None):
        self._state.reseed(seed)

    def random(self, size=None):
        return self._state.random(size)

    random_sample = random

    def rand(self, *shape):
        return self._state.random(shape if shape else None)

    def randn(self, *shape):
        return self._state.standard_normal(shape if shape else None)

    def uniform(self, low=0.0, high=1.0, size=None):
        return self._state.uniform(low, high, size)

    def normal(self, loc=0.0, scale=1.0, size=None):
        return self._state.normal(loc, scale, size)

    def standard_normal(self, size=None):
        return self._state.standard_normal(size)

    def randint(self, low, high=None, size=None, dtype=np.int64):
        return self._state.integers(low, high, size, dtype)

    def choice(self, a, size=None, replace=True, p=None):
        return self._state.choice(a, size, replace, p)

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        raise NotImplementedError("ramba_b200.random.RandomState.%s is not implemented (supported: %s)"
                                  % (name, ", ".join(sorted(self._METHODS))))
