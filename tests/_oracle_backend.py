"""TEST-ONLY: run the engine's op lists through the NumPy oracle on host buffers, so that the
fuser / partitioner / exchange logic can be exercised without a GPU.  The product never does
this (ramba_b200.runtime raises without CUDA).  Op lists go through the oracle extended by the
PHILOX draws (_philox_vm); gather, scatter, route and the grouped reduction through the NumPy
restatements of those kernels (_index_vm, _group_vm)."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


PLANS = []     # rb200_describe_plan() of every op list handed to the executor (which kernel the CUDA library would run)
REJECTED = []  # (message, op list summary) of every op list the CUDA library's validation refused


def _library_accepts(fop):
    """Hand the op list to the real library's validation as well (CPU only: it validates the op list before it looks
    for a device, and never touches the pointers).  Anything but 'no usable CUDA device' means the oracle executes
    something the CUDA library would refuse."""
    import ctypes as C

    from ramba_b200 import _cabi

    try:
        lib = _cabi.load()
    except _cabi.CabiError:
        return  # library not built: test_cabi_exports complains about that
    import torch

    if torch.cuda.is_available():
        return  # with a device present the call would launch on host pointers
    rc = lib.rb200_run_deferred_ops(C.byref(fop), None)
    msg = lib.rb200_last_error().decode() if rc != 0 else ""
    if rc != 0 and "no usable CUDA device" not in msg:
        REJECTED.append((msg, "ndim=%d n_views=%d n_insns=%d n_regs=%d" % (fop.ndim, fop.n_views, fop.n_insns, fop.n_regs)))
        raise AssertionError("libramba_b200 would reject this op list: " + msg)


class OracleBackend:
    """Stands where ramba_b200.runtime.CudaBackend does: op lists are evaluated by the NumPy oracle on host buffers, ranks
    talk over gloo.  Lives in the test package; the product has no reference to it."""

    name = "oracle"
    dist_backend = "gloo"
    timing = False

    def __init__(self):
        import torch

        import _philox_vm

        self.device = torch.device("cpu")
        self.reduce_partials = _philox_vm.reduce_partials
        self._vm = _philox_vm

    def run(self, fop, stream=None):
        _library_accepts(fop)
        try:
            from ramba_b200 import _cabi

            PLANS.append(_cabi.describe_plan(fop))
        except Exception as ex:  # library not built: test_cabi_exports complains about that
            PLANS.append("unavailable: %s" % (ex,))
        return self._vm.run_deferred_ops(fop, stream)

    def stream_handle(self):
        return None

    def red_scratch_bytes(self):
        from ramba_b200 import _cabi

        return 256 + 8 * _cabi.MAX_REDS * 4096

    def cumulative(self, src_ptr, dst_ptr, code, n_outer, length, n_inner, redop, carry_in, totals_out):
        self._vm.cumulative(src_ptr, dst_ptr, code, n_outer, length, n_inner, redop, carry_in, totals_out, None, None)
        return None

    def gather(self, view, lin, n, out, bad):
        import _index_vm

        _index_vm.gather(view, lin, n, out, bad)

    def scatter(self, view, lin, n, values, bad):
        import _index_vm

        _index_vm.scatter(view, lin, n, values, bad)

    def route(self, table, lin, n, offsets, slots, counts, bad):
        import _index_vm

        _index_vm.route(table, lin, n, offsets, slots, counts, bad)
        return None

    def group_reduce(self, view, src_code, axis, table, op, center, out):
        import _group_vm

        _group_vm._library_accepts(view, src_code, axis, table, op, center, out)
        _group_vm.group_reduce(view, src_code, axis, table, op, center, out)
        return None

    def init_process_group(self):
        import torch.distributed as dist

        dist.init_process_group("gloo")

    def synchronize(self):
        pass


def install():
    from ramba_b200.runtime import RT

    RT.backend = OracleBackend()
