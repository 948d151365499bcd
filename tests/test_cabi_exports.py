"""The C-ABI library loads (no GPU needed) and exports every symbol include/ramba_b200.h declares;
without a CUDA device launches fail loudly instead of falling back."""
import ctypes
import os
import re

import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")


def test_library_exports_header_symbols():
    from ramba_b200 import _cabi

    hdr = open(os.path.join(ROOT, "include", "ramba_b200.h")).read()
    declared = set(re.findall(r"\b(rb200_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(_cabi.EXPORTS), (declared, set(_cabi.EXPORTS))
    lib = ctypes.CDLL(_cabi.lib_path())
    for name in declared:
        assert hasattr(lib, name), name
    assert _cabi.load().rb200_abi_version() == _cabi.ABI_VERSION


def test_struct_layout_matches_header(tmp_path):
    """sizeof / offsetof of every struct as gcc sees include/ramba_b200.h == the ctypes mirror in _cabi.py."""
    import subprocess

    from ramba_b200 import _cabi

    src = tmp_path / "layout.c"
    src.write_text(r"""
#include <stdio.h>
#include <stddef.h>
#include "ramba_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu\n", sizeof(rb200_insn), sizeof(rb200_view), sizeof(rb200_red), sizeof(rb200_fused_op));
  printf("%zu %zu %zu %zu %zu\n", offsetof(rb200_view, stride), offsetof(rb200_view, dtype), offsetof(rb200_view, alloc_lo),
         offsetof(rb200_fused_op, views), offsetof(rb200_fused_op, insns));
  printf("%zu %zu %zu %d %d\n", offsetof(rb200_fused_op, scalars), offsetof(rb200_fused_op, reds), offsetof(rb200_fused_op, red_scratch),
         RB200_ABI_VERSION, RB200_NUM_OPS);
  return 0;
}
""")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)]).decode().split()
    got = [int(x) for x in out]
    F = _cabi.FusedOp
    exp = [ctypes.sizeof(_cabi.Insn), ctypes.sizeof(_cabi.View), ctypes.sizeof(_cabi.Red), ctypes.sizeof(F),
           _cabi.View.stride.offset, _cabi.View.dtype.offset, _cabi.View.alloc_lo.offset, F.views.offset, F.insns.offset,
           F.scalars.offset, F.reds.offset, F.red_scratch.offset, _cabi.ABI_VERSION, len(_cabi.OPS)]
    assert got == exp
    assert ctypes.sizeof(_cabi.Insn) == 16


def test_no_cpu_fallback_without_cuda():
    import torch

    if torch.cuda.is_available():
        pytest.skip("needs a machine without a GPU")
    from ramba_b200 import _cabi

    fop = _cabi.FusedOp()
    fop.abi_version = _cabi.ABI_VERSION
    fop.ndim = 1
    fop.itershape[0] = 16
    fop.n_insns = 1
    with pytest.raises(_cabi.CabiError):
        _cabi.run_deferred_ops(fop)
    from ramba_b200.runtime import Runtime

    with pytest.raises(RuntimeError):
        Runtime().device


def _one_insn_op():
    """A minimal well-formed fused op: views[0][0:10] = scalars[0] (float64)."""
    from ramba_b200 import _cabi

    f = _cabi.FusedOp()
    f.abi_version = _cabi.ABI_VERSION
    f.ndim, f.n_views, f.n_insns, f.n_scalars, f.num_workers = 1, 1, 1, 1, 1
    f.itershape[0] = 10
    f.views[0].base = 0x1000  # never dereferenced: every case below is rejected (or empty) before a launch
    f.views[0].stride[0] = 1
    f.views[0].dtype = _cabi.F64
    i = f.insns[0]
    i.op, i.ctype, i.a_kind, i.a_idx = _cabi.OP["MOV"], _cabi.T_F64, _cabi.K_SCAL, 0
    i.st_reg = i.st2 = i.mask_reg = _cabi.NOSTORE
    i.st_view = 0
    return f


def _null_reduction_output(f):
    """A global reduction whose reds[0].out is null."""
    from ramba_b200 import _cabi

    f.n_reds = 1
    f.red_scratch = 0x2000
    f.reds[0].op, f.reds[0].ctype, f.reds[0].out_dtype = _cabi.RED_ADD, _cabi.T_F64, _cabi.F64


def test_malformed_op_lists_are_rejected_with_a_reason():
    """Error convention of the boundary (include/ramba_b200.h): nonzero status + thread-local message; the op
    list is validated before any device work, so this needs no GPU.  rb200_describe_plan validates the same way."""
    import ctypes as C

    from ramba_b200 import _cabi

    lib = _cabi.load()

    def run(mutate):
        f = _one_insn_op()
        mutate(f)
        rc = lib.rb200_run_deferred_ops(C.byref(f), None)
        return rc, lib.rb200_last_error().decode()

    def describe(mutate):
        f = _one_insn_op()
        mutate(f)
        buf = C.create_string_buffer(600)
        rc = lib.rb200_describe_plan(C.byref(f), buf, 600)
        return rc, (lib.rb200_last_error() if rc else buf.value).decode()

    cases = [
        (lambda f: setattr(f, "abi_version", 99), "ABI version"),
        (lambda f: setattr(f, "ndim", 9), "ndim"),
        (lambda f: setattr(f, "n_insns", 500), "too many instructions"),
        (lambda f: f.itershape.__setitem__(0, -1), "negative itershape"),
        (lambda f: setattr(f.insns[0], "op", 200), "bad opcode"),
        (lambda f: setattr(f.insns[0], "ctype", 7), "bad compute class"),
        (lambda f: setattr(f.insns[0], "a_kind", 9), "bad operand kind"),
        (lambda f: setattr(f.insns[0], "a_idx", 5), "scalar index out of range"),
        (lambda f: setattr(f.insns[0], "st_view", 3), "st_view out of range"),
        (lambda f: setattr(f.insns[0], "st_reg", 2), "st_reg out of range"),
        (lambda f: setattr(f.insns[0], "mask_reg", 1), "mask_reg out of range"),
        (lambda f: setattr(f.views[0], "dtype", 55), "bad view dtype"),
        (lambda f: setattr(f.views[0], "base", 0), "null view base pointer"),
        (_null_reduction_output, "null reduction output"),
    ]
    for mutate, reason in cases:
        for call in (run, describe):
            rc, msg = call(mutate)
            assert rc != 0 and reason in msg, (call.__name__, reason, rc, msg)
    # an empty iteration space is a successful no-op
    rc, _ = run(lambda f: f.itershape.__setitem__(0, 0))
    assert rc == 0
    assert describe(lambda f: f.itershape.__setitem__(0, 0)) == (0, "kernel=none")
    with pytest.raises(_cabi.CabiError):
        bad = _one_insn_op()
        bad.insns[0].op = 200
        _cabi.run_deferred_ops(bad)


def test_cuda_backend_wiring(monkeypatch):
    """The one backend of the package (ramba_b200.runtime.CudaBackend) with the torch.cuda calls it makes replaced by fakes:
    the library is loaded, op lists go to rb200_run_deferred_ops, partial folds to rb200_reduce_partials, ranks talk NCCL."""
    import torch

    from ramba_b200 import _cabi, runtime

    class FakeStream:
        cuda_stream = 1234

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: FakeStream())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda d=None: None)
    be = runtime.CudaBackend()
    assert be.device.type == "cuda" and be.stream_handle() == 1234 and be.dist_backend == "nccl" and be.timing
    assert be.run is _cabi.run_deferred_ops and be.reduce_partials is _cabi.reduce_partials
    assert be.red_scratch_bytes() == _cabi.red_scratch_bytes() > 0
    be.synchronize()
    rt = runtime.Runtime()
    rt.backend = be
    assert rt.is_cuda and rt.device == be.device and rt.executor() is _cabi.run_deferred_ops
