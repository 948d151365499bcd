"""TEST-ONLY: RB200_OP_PHILOX restated in NumPy from its contract (include/ramba_b200.h), written independently of the CUDA
code, plus an op-list evaluator that runs op lists containing PHILOX instructions through the NumPy oracle
(oracle/vm.py) on host buffers.

The oracle evaluates whole op lists at once; it knows every opcode but PHILOX.  `run_deferred_ops` evaluates each PHILOX
instruction here and hands the oracle an op list in which it has become a load of the values computed:
  1. the index operand is evaluated by running the instructions before it (without their stores and reductions) plus
     one MOV of the operand into a temporary int64 view;
  2. the draw is computed from those indices;
  3. the PHILOX instruction becomes a MOV from a temporary view holding the draw, keeping its register / view stores.
The index of a draw is arithmetic on IOTA operands, which step 1 reproduces exactly.
"""
import types

import numpy as np

from oracle import vm

PHILOX = 55
UNIFORM64, UNIFORM32, NORMAL64, INTEGER = range(4)
M32 = np.uint64(0xFFFFFFFF)
_U = np.uint64


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on arrays of 32-bit words held in uint64 (Salmon et al., SC'11): returns (w0, w1, w2, w3)."""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint64) & M32 for x in (c0, c1, c2, c3))
    k0, k1 = np.asarray(k0, dtype=np.uint64) & M32, np.asarray(k1, dtype=np.uint64) & M32
    for r in range(10):
        if r:
            k0 = (k0 + _U(0x9E3779B9)) & M32
            k1 = (k1 + _U(0xBB67AE85)) & M32
        p0 = _U(0xD2511F53) * c0
        p1 = _U(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> _U(32)) ^ c1 ^ k0, p1 & M32, (p0 >> _U(32)) ^ c3 ^ k1, p0 & M32
    return c0, c1, c2, c3


def block(j, key):
    """Words of the block with number j (uint64 array) of the draw with 64-bit key `key`."""
    j = np.asarray(j, dtype=np.uint64)
    key = _U(int(key) & 0xFFFFFFFFFFFFFFFF)
    return philox4x32_10(j & M32, j >> _U(32), np.zeros_like(j), np.zeros_like(j), key & M32, key >> _U(32))


def mulhi64(x, n):
    """High 64 bits of the 128-bit product x * n, from 32-bit halves."""
    x = np.asarray(x, dtype=np.uint64)
    n = _U(int(n))
    xl, xh, nl, nh = x & M32, x >> _U(32), n & M32, n >> _U(32)
    ll, lh, hl, hh = xl * nl, xl * nh, xh * nl, xh * nh
    mid = (ll >> _U(32)) + (lh & M32) + (hl & M32)
    return hh + (lh >> _U(32)) + (hl >> _U(32)) + (mid >> _U(32))


def _u01_64(x):
    return (x >> _U(11)).astype(np.float64) * 2.0 ** -53


def draw(i, key, form, bound=1):
    """Values of elements with linear indices `i` (int64 array) of a draw."""
    u = np.asarray(i, dtype=np.int64).astype(np.uint64)
    if form == UNIFORM32:
        w = block(u >> _U(2), key)
        lane = (u & _U(3)).astype(np.int64)
        x = np.choose(lane, w)
        return (x >> _U(8)).astype(np.float32) * np.float32(2.0 ** -24)
    w0, w1, w2, w3 = block(u >> _U(1), key)
    odd = (u & _U(1)) != 0
    x0 = w0 | (w1 << _U(32))
    x1 = w2 | (w3 << _U(32))
    if form == NORMAL64:
        u1 = 1.0 - _u01_64(x0)
        u2 = _u01_64(x1)
        r = np.sqrt(-2.0 * np.log(u1))
        t = (2.0 * np.pi) * u2
        return np.where(odd, r * np.sin(t), r * np.cos(t))
    x = np.where(odd, x1, x0)
    if form == INTEGER:
        return mulhi64(x, bound).astype(np.int64)
    return _u01_64(x)


_CLS = {UNIFORM64: (vm.T_F64, vm.F64, np.float64), UNIFORM32: (vm.T_F32, vm.F32, np.float32),
        NORMAL64: (vm.T_F64, vm.F64, np.float64), INTEGER: (vm.T_I64, vm.I64, np.int64)}
_INSN_FIELDS = ("op", "ctype", "a_kind", "a_idx", "b_kind", "b_idx", "c_kind", "c_idx", "st_reg", "st_view", "st2", "mask_reg",
                "imm")


def _insn(I, **kw):
    d = {f: getattr(I, f) for f in _INSN_FIELDS}
    d.update(kw)
    return types.SimpleNamespace(**d)


def _view(base, code, shape):
    st, s = [], 1
    for n in reversed(shape):
        st.append(s)
        s *= n
    st = list(reversed(st)) + [0] * (5 - len(shape))
    return types.SimpleNamespace(base=base, stride=st, dtype=code, flags=0, alloc_lo=None, alloc_hi=None)


def _copy(fop):
    ns = types.SimpleNamespace()
    for f in ("ndim", "worker_num", "num_workers", "n_views", "n_scalars", "n_insns", "n_regs", "n_reds", "n_axis_red_dims",
              "axis_nsplit", "red_scratch", "abi_version"):
        setattr(ns, f, getattr(fop, f))
    ns.itershape = list(fop.itershape)
    ns.global_start = list(fop.global_start)
    ns.views = [fop.views[i] for i in range(fop.n_views)]
    ns.scalars = list(fop.scalars)
    ns.insns = [_insn(fop.insns[i]) for i in range(fop.n_insns)]
    ns.reds = [fop.reds[i] for i in range(len(fop.reds))]
    return ns


def run_deferred_ops(fop, stream=None):
    """oracle.vm.run_deferred_ops, extended by PHILOX."""
    if not any(fop.insns[i].op == PHILOX for i in range(fop.n_insns)):
        return vm.run_deferred_ops(fop, stream)
    nd = fop.ndim
    shape = tuple(int(fop.itershape[d]) for d in range(nd))
    if any(s == 0 for s in shape) or fop.n_insns == 0:
        return
    ns = _copy(fop)
    keep = []  # temporaries stay alive until the oracle has run
    for pc in range(ns.n_insns):
        I = ns.insns[pc]
        if I.op != PHILOX:
            continue
        # 1. the index operand, from the side-effect free prefix
        pre = _copy(fop)
        pre.views = list(ns.views)
        pre.insns = []
        for J in ns.insns[:pc]:
            if J.op == vm.OPS.index("RED"):
                continue
            pre.insns.append(_insn(J, st_view=vm.NOSTORE, mask_reg=vm.NOSTORE,
                                   c_kind=vm.K_NONE if J.op == vm.OPS.index("SINCOS") else J.c_kind))
        idx = np.zeros(shape, dtype=np.int64)
        keep.append(idx)
        pre.views.append(_view(idx.ctypes.data, vm.I64, shape))
        pre.insns.append(types.SimpleNamespace(op=vm.OPS.index("MOV"), ctype=vm.T_I64, a_kind=I.a_kind, a_idx=I.a_idx, b_kind=vm.K_NONE,
                                               b_idx=0, c_kind=vm.K_NONE, c_idx=0, st_reg=vm.NOSTORE, st_view=len(pre.views) - 1,
                                               st2=vm.NOSTORE, mask_reg=vm.NOSTORE, imm=0))
        pre.n_views, pre.n_insns, pre.n_reds = len(pre.views), len(pre.insns), 0
        vm.run_deferred_ops(pre)
        # 2. the draw
        cls, code, dt = _CLS[I.imm]
        key = int(ns.scalars[I.b_idx])
        bound = int(np.uint64(ns.scalars[I.c_idx]).astype(np.int64)) if I.imm == INTEGER else 1
        vals = np.ascontiguousarray(draw(idx, key, I.imm, bound).astype(dt))
        keep.append(vals)
        ns.views.append(_view(vals.ctypes.data, code, shape))
        # 3. PHILOX -> MOV from the draw
        ns.insns[pc] = _insn(I, op=vm.OPS.index("MOV"), ctype=cls, a_kind=vm.K_VIEW, a_idx=len(ns.views) - 1, b_kind=vm.K_NONE,
                             b_idx=0, c_kind=vm.K_NONE, c_idx=0, imm=0)
    ns.n_views = len(ns.views)
    vm.run_deferred_ops(ns, stream)
    del keep


reduce_partials = vm.reduce_partials
cumulative = vm.cumulative
