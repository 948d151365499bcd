"""ramba_b200 — H100-native drop-in for the fused elementwise / reduction / shifted-slice hot path
of Python-for-HPC/ramba (`import ramba_b200 as np`).

Mirrors ramba/__init__.py:13-19: re-exports the array API of `ramba_b200.ramba` plus the NumPy
dtypes.  Execution goes through libramba_b200.so (hand-written sm_90a kernels) — there is no
CPU path.
"""
from numpy import (bool_, byte, double, dtype, e, float16, float32, float64, half, iinfo, finfo, inf, int8, int16, int32, int64, int_,  # noqa: F401
                   intc, longlong, nan, newaxis, pi, short, single, ubyte, uint, uint8, uint16, uint32, uint64, uintc, ulonglong, ushort)

from . import common  # noqa: F401
from .ramba import *  # noqa: F401,F403
from .ramba import (ndarray, bdarray, deferred_op, sync, arange, empty, zeros, ones, full, fromarray, fromfunction,  # noqa: F401
                    asarray, array, where, HANDLED_FUNCTIONS, fromarray_local, local_block_to_host, stencil, sstencil)
from . import ramba as _ramba
from . import random  # noqa: F401  (`import ramba_b200.random as random`, like ramba.random)

globals().update(_ramba.api)  # abs/min/max/sum/all/any shadow the builtins like in the reference

__version__ = "0.1.0"
