"""Worker runtime: this rank's shards in HBM and the execution of fused ops on them.

Stands where RemoteState does in the reference (ramba/ramba.py:1880-3971), for ONE worker — the
process's own GPU.  The driver/worker RPC layer (ramba/ramba.py:3985-4104) disappears: under SPMD
every rank runs the driver and calls its own runtime directly.

  * shards: one flat torch tensor per (gid) holding this worker's block, allocated lazily at the
    first flush that touches it (ramba/ramba.py:3506-3523, 1947-2005) and freed when the last
    handle dies (destroy_array, ramba/ramba.py:1943-1945);
  * launch: binds an op list to one range and calls the C-ABI (ramba/ramba.py:3758-3780);
  * transfers: grouped NCCL send / receive, all-gather, all-reduce and broadcast instead of pickled
    mailbox messages (ramba/ramba.py:3646-3693), each counted in bytes_sent / collectives by one rule.

PyTorch is used for device memory, streams and torch.distributed only.
"""
import ctypes
import os

import numpy as np
import torch
import torch.distributed as dist

from . import _cabi as cabi
from . import common
from . import shardview
from .program import REDUCTIONS, np_dtype, rb_dtype

_TORCH_DTYPE = {
    np.dtype(np.float64): torch.float64,
    np.dtype(np.float32): torch.float32,
    np.dtype(np.int64): torch.int64,
    np.dtype(np.int32): torch.int32,
    np.dtype(np.bool_): torch.uint8,  # stored as bytes 0/1
    np.dtype(np.uint8): torch.uint8,
    np.dtype(np.int8): torch.int8,
    np.dtype(np.int16): torch.int16,
    np.dtype(np.uint16): torch.uint16,
    np.dtype(np.uint32): torch.uint32,
}


def torch_dtype(dt):
    return _TORCH_DTYPE[np.dtype(dt)]


class Shard:
    """This worker's block of one bdarray (LocalNdarray, ramba/ramba.py:1169-1357).  With `border` > 0 the buffer is the
    block grown by `border` elements on every side of every dim (`np.empty(dim_lens + 2*border)`,
    ramba/ramba.py:1208-1214): the ring receives the neighbours' edge elements (getborder,
    ramba/ramba.py:1260-1322), so that shifted views of the array read ONE buffer with ONE set of strides."""

    __slots__ = ("buf", "shape", "dtype", "strides", "bounds", "border", "origin")

    _layouts = {}  # (shape, border) -> (strides, origin): a pure function, asked for every new result array

    def __init__(self, buf, shape, dtype, border=0):
        self.buf = buf
        shape = self.shape = tuple([int(s) for s in shape])
        self.dtype = np.dtype(dtype)
        border = self.border = int(border)
        self.strides, self.origin = Shard.layout(shape, border)  # origin: element offset of interior element (0, 0, ...)
        p = buf.data_ptr()
        self.bounds = (p, p + buf.numel() * buf.element_size())  # [alloc_lo, alloc_hi) handed to the C-ABI

    @staticmethod
    def layout(shape, border):
        """(element strides, origin) of a block of `shape` grown by `border`: also what another rank's shard looks like."""
        lay = Shard._layouts.get((shape, border))
        if lay is None:
            st = []
            acc = 1
            for s in reversed(shape):
                st.append(acc)
                acc *= max(1, s + 2 * border)
            strides = tuple(reversed(st))  # elements, C order over the padded block
            if len(Shard._layouts) >= 4096:
                Shard._layouts.clear()
            lay = Shard._layouts[(shape, border)] = (strides, sum(border * x for x in strides))
        return lay

    def ptr(self, off=0):
        """Device address of interior-relative element offset `off`."""
        return self.buf.data_ptr() + (self.origin + off) * self.dtype.itemsize

    def interior(self):
        """torch view of the block without its ring (contiguous when border == 0)."""
        n = 1
        for x in self.shape:
            n *= x
        if self.border == 0:
            return self.buf[:n].view(self.shape) if self.shape else self.buf[:1]
        return self.buf.as_strided(self.shape, self.strides, self.origin)


class CudaBackend:
    """Where op lists run: libramba_b200.so on this process's GPU, NCCL between the processes.  It is the only backend the
    package has; `Runtime.backend` is an attribute so that the test package can put its own object there (the oracle on
    host buffers, tests/_oracle_backend.py) - nothing in the product refers to, constructs or imports another one."""

    name = "cuda"
    dist_backend = "nccl"
    timing = True  # CUDA events around launches (bench.py's per-kernel times)

    def __init__(self):
        cabi.load()  # raises if the library is missing: there is no fallback
        if not torch.cuda.is_available():
            raise RuntimeError(
                "ramba_b200 needs a CUDA device (H100, sm_90a): torch.cuda.is_available() is False and "
                "there is no CPU execution path")
        self.device = torch.device("cuda", common.local_rank)
        torch.cuda.set_device(self.device)
        self.run = cabi.run_deferred_ops
        self.reduce_partials = cabi.reduce_partials

    def stream_handle(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def red_scratch_bytes(self):
        return cabi.red_scratch_bytes()

    def cumulative(self, src_ptr, dst_ptr, code, n_outer, length, n_inner, redop, carry_in, totals_out):
        """rb200_cumulative on the current stream; returns the scratch buffer (the caller keeps it alive)."""
        nbytes = cabi.cumulative_scratch_bytes(n_outer, length, n_inner)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        cabi.cumulative(src_ptr, dst_ptr, code, n_outer, length, n_inner, redop, carry_in, totals_out, scratch.data_ptr(),
                        self.stream_handle())
        return scratch

    def gather(self, view, lin, n, out, bad):
        """rb200_gather on the current stream: out[i] = view[lin[i]] (view: a cabi.IndexView)."""
        cabi.gather(view, lin, n, out, bad, self.stream_handle())

    def scatter(self, view, lin, n, values, bad):
        """rb200_scatter on the current stream: view[lin[i]] = values[i]."""
        cabi.scatter(view, lin, n, values, bad, self.stream_handle())

    def route(self, table, lin, n, offsets, slots, counts, bad):
        """rb200_route on the current stream; returns the scratch buffer (the caller keeps it alive)."""
        scratch = torch.empty(cabi.route_scratch_bytes(n, table.n_ranks), dtype=torch.uint8, device=self.device)
        cabi.route(table, lin, n, offsets, slots, counts, bad, scratch.data_ptr(), self.stream_handle())
        return scratch

    def group_reduce(self, view, src_code, axis, table, op, center, out):
        """rb200_group_reduce on the current stream; returns the scratch buffer (the caller keeps it alive)."""
        nbytes = cabi.group_reduce_scratch_bytes(view, axis, table.n_groups)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device) if nbytes else None
        cabi.group_reduce(view, src_code, axis, table, op, center, out, scratch.data_ptr() if nbytes else None, self.stream_handle())
        return scratch

    def arg_reduce(self, view, src_code, axis, op, origin, gstride, out_idx, out_key):
        """rb200_arg_reduce on the current stream; returns the scratch buffer (the caller keeps it alive)."""
        nbytes = cabi.arg_reduce_scratch_bytes(view, axis)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device) if nbytes else None
        o, g = cabi.arg_coords(origin, gstride)
        cabi.arg_reduce(view, src_code, axis, op, o, g, out_idx, out_key, scratch.data_ptr() if nbytes else None, self.stream_handle())
        return scratch

    def compact_count(self, cond, cond_code, run_len, counts):
        """rb200_compact_count on the current stream."""
        cabi.compact_count(cond, cond_code, run_len, counts, self.stream_handle())

    def compact(self, cond, cond_code, run_len, counts, incl, run_base, form, values, origin, gstride, outs):
        """rb200_compact on the current stream."""
        cabi.compact(cond, cond_code, run_len, counts, incl, run_base, form, values, origin, gstride, outs, self.stream_handle())

    def histogram(self, view, src_code, wview, w_code, table, out, bad):
        """rb200_histogram on the current stream; returns the scratch buffer (the caller keeps it alive)."""
        nbytes = cabi.histogram_scratch_bytes(view, wview is not None, table)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device) if nbytes else None
        cabi.histogram(view, src_code, wview, w_code, table, out, bad, scratch.data_ptr() if nbytes else None, self.stream_handle())
        return scratch

    def bin_search(self, view, src_code, sorted_ptr, n_sorted, sorted_code, side, out):
        """rb200_bin_search on the current stream."""
        cabi.bin_search(view, src_code, sorted_ptr, n_sorted, sorted_code, side, out, self.stream_handle())

    def select_count(self, view, src_code, seg_len, state, pass_, mode):
        """rb200_select_count on the current stream."""
        cabi.select_count(view, src_code, seg_len, state, pass_, mode, self.stream_handle())

    def select_choose(self, view, src_code, seg_len, state, pass_):
        """rb200_select_choose on the current stream."""
        cabi.select_choose(view, src_code, seg_len, state, pass_, self.stream_handle())

    def select_rows(self, view, src_code, seg_len, targets, rank_table, skip_nan, keys, nans):
        """rb200_select_rows on the current stream."""
        cabi.select_rows(view, src_code, seg_len, targets, rank_table, skip_nan, keys, nans, self.stream_handle())

    def init_process_group(self):
        dist.init_process_group("nccl", device_id=self.device)

    def synchronize(self):
        torch.cuda.synchronize(self.device)

    def events(self):
        return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


class Runtime:
    def __init__(self):
        self.shards = {}
        self.backend = None  # CudaBackend(), made at first use
        self._red_scratch = None
        self._pg_ready = False
        self.launches = 0
        self.bytes_sent = 0
        self.collectives = 0  # all-gather / all-reduce / broadcast calls issued
        self.ring_receives = 0  # halo pieces received into the ring of a padded block (getborder)
        self.held = ()  # see hold()
        self.profile_events = None  # list -> (start, end, n_insns) CUDA events around every launch
        self.on_reset = []  # the engine registers what else must be forgotten with the shards (pending DAG nodes, fused op)

    # ---- backend / device / process group --------------------------------------------------
    def be(self):
        b = self.backend
        if b is None:
            b = self.backend = CudaBackend()
        return b

    @property
    def device(self):
        return self.be().device

    @property
    def is_cuda(self):
        """True when op lists go to the CUDA library (always, outside the test package)."""
        return isinstance(self.be(), CudaBackend)

    def reset(self):
        """Forget every shard (and whatever the engine registered in on_reset); the next use builds the CUDA backend."""
        for hook in self.on_reset:
            hook()
        self.shards.clear()
        self.backend = None
        self._red_scratch = None

    def executor(self):
        return self.be().run

    def hold(self, *objs):
        """Keep objs alive until the next hold: buffers that launches or transfers already enqueued on the current stream
        still use.  Holding them is enough because the caching allocator hands a freed buffer out again in stream order;
        a buffer that something not yet enqueued will read needs another owner.  Each hold replaces the last one (sync()
        leaves them alone), so what is held never grows."""
        self.held = objs

    def ensure_process_group(self):
        if common.num_workers <= 1 or self._pg_ready:
            return
        if not dist.is_initialized():
            self.be().init_process_group()
        self._pg_ready = True

    # ---- transfers between ranks: the only code of the package that talks to other ranks.  Counting rule (DESIGN.md §4):
    # a grouped send / receive adds the bytes of every send; an all-gather adds one collective and the bytes of this rank's
    # part times W-1; an all-reduce one collective and the bytes of the tensor; a broadcast one collective and, on the
    # source rank, the bytes of the tensor times W-1.
    def p2p(self, ops):
        """ops: [(is_send, tensor, peer)] -> the works of ONE grouped send / receive of their bytes, not waited for."""
        if not ops:
            return []
        self.ensure_process_group()
        pending = []
        for is_send, t, peer in ops:
            if is_send:
                self.bytes_sent += t.numel() * t.element_size()
            pending.append(dist.P2POp(dist.isend if is_send else dist.irecv, t.view(torch.uint8), peer))
        return dist.batch_isend_irecv(pending)

    def all_gather(self, full, mine):
        """Every rank's `mine`, in rank order, into `full`; returns the work, not waited for."""
        self.ensure_process_group()
        self.collectives += 1
        self.bytes_sent += mine.numel() * mine.element_size() * (common.num_workers - 1)
        return dist.all_gather_into_tensor(full.view(torch.uint8), mine.view(torch.uint8), async_op=True)

    def all_reduce(self, t, op):
        """t = op over every rank's t, in place; op: sum prod min max all any."""
        self.ensure_process_group()
        self.collectives += 1
        self.bytes_sent += t.numel() * t.element_size()
        dist.all_reduce(t, op=getattr(dist.ReduceOp, REDUCTIONS[op].allreduce))

    def broadcast(self, t, src):
        """Rank src's t into every rank's t, in place."""
        self.ensure_process_group()
        self.collectives += 1
        if common.worker_num == src:
            self.bytes_sent += t.numel() * t.element_size() * (common.num_workers - 1)
        dist.broadcast(t, src=src)

    # ---- shard storage --------------------------------------------------------------------
    def create_array(self, gid, local_shape, dtype, border=0):
        """Allocate this worker's block (uninitialised, like np.empty at ramba/ramba.py:1208-1214), grown by `border` on
        every side when the array was created with local_border."""
        if gid in self.shards:
            return self.shards[gid]
        n = 1
        for s in local_shape:
            n *= int(s)
        if n == 0:
            border = 0
        if border:
            n = 1
            for s in local_shape:
                n *= int(s) + 2 * border
        buf = torch.empty(max(n, 1), dtype=torch_dtype(dtype), device=self.device)
        if border:
            buf.zero_()  # the ring of a block at the array's edge is never received: keep it defined
        sh = Shard(buf, local_shape, dtype, border)
        self.shards[gid] = sh
        return sh

    def destroy_array(self, gid):
        self.shards.pop(gid, None)

    def red_scratch(self):
        if self._red_scratch is None:
            nbytes = self.be().red_scratch_bytes()
            self._red_scratch = torch.zeros(nbytes // 8 + 1, dtype=torch.int64, device=self.device)
        return self._red_scratch

    # ---- view binding -----------------------------------------------------------------------
    @staticmethod
    def bind_view(sv, local_strides, rng):
        """(element offset, per-iteration-dim element strides) of view part `sv` (this worker's
        shardview of the view) for iteration range `rng` (clean box inside sv's box), given the
        C-order strides of the local buffer."""
        k = len(sv.size)
        off = 0
        used = set()
        strides = [0] * k
        for d in range(k):
            a = int(sv.axis_map[d])
            if a < 0:
                continue
            used.add(a)
            i0 = int(rng.start[d] - sv.start[d])
            st = int(sv.steps[d])
            if st > 0:
                coord = int(sv.base_offset[a]) + i0 * st
            else:
                coord = int(sv.base_offset[a]) + (int(sv.size[d]) - 1 - i0) * (-st)
            off += coord * local_strides[a]
            strides[d] = st * local_strides[a]
        for a in range(len(sv.base_offset)):
            if a not in used:
                off += int(sv.base_offset[a]) * local_strides[a]
        return off, strides

    # ---- launching ----------------------------------------------------------------------------
    def launch(self, *args, **kw):
        """submit(bind(...)): bind an op list to one range and hand it to the C-ABI."""
        return self.submit(self.bind(*args, **kw))

    def bind(self, program, rng_shape, gstart, bound_views, reds=None, n_axis_red=0, axis_nsplit=1,
             axis_partials=None, worker_num=0, num_workers=1):
        """Bind `program` to one range: the rb200_fused_op to submit.
        bound_views: list of (data_ptr, elem strides per iteration dim, rb dtype)."""
        # ---- launch memo: everything in the bound struct except the addresses is a function of (op list, range, strides)
        key = (program, tuple([int(s) for s in rng_shape]), tuple([int(g) for g in gstart]),
               tuple([(tuple(bv[1]), bv[2], len(bv) > 3 and bv[3] is not None) for bv in bound_views]),
               None if reds is None else tuple([None if r is None else r[1] for r in reds]),
               n_axis_red, axis_nsplit, worker_num, num_workers)
        tpl = _launch_cache.get(key)
        if tpl is not None:
            outs = scratch = None
            if program.reds:
                if reds is not None:
                    outs = [None if r is None else r[0] for r in reds]
                scratch = axis_partials if n_axis_red else self.red_scratch().data_ptr()
            fop = fill_template(tpl, [(bv[0], bv[3] if len(bv) > 3 else None) for bv in bound_views], outs, scratch)
            if _VERIFY_PLAN_CACHE:
                fresh = self._build(program, rng_shape, gstart, bound_views, reds, n_axis_red, axis_nsplit, axis_partials, worker_num, num_workers)
                if ctypes.string_at(ctypes.addressof(fop), ctypes.sizeof(fop)) != ctypes.string_at(ctypes.addressof(fresh), ctypes.sizeof(fresh)):
                    raise AssertionError("launch memo: the patched template differs from a freshly bound op list")
        else:
            fop = self._build(program, rng_shape, gstart, bound_views, reds, n_axis_red, axis_nsplit, axis_partials, worker_num, num_workers)
            if len(_launch_cache) >= 4096:
                _launch_cache.clear()
            _launch_cache[key] = ctypes.string_at(ctypes.addressof(fop), ctypes.sizeof(fop))
        return fop

    def _build(self, program, rng_shape, gstart, bound_views, reds, n_axis_red, axis_nsplit, axis_partials, worker_num, num_workers):
        """Fill one rb200_fused_op from scratch (collapse / merge the iteration dims, copy the op list, bind the views)."""
        ndim = len(rng_shape)
        dims = list(range(ndim))
        shape = [int(s) for s in rng_shape]
        strides = [list(bv[1]) for bv in bound_views]
        gs = [int(g) for g in gstart]
        iota_dims = set(program.uses_iota)
        # --- collapse: drop extent-1 dims, merge dims that are contiguous for every view
        red_dims = set(range(n_axis_red))
        keep = [d for d in dims if shape[d] != 1 or d in iota_dims]
        if n_axis_red and not any(d in red_dims for d in keep):
            keep = [0] + keep
        if not any(d not in red_dims for d in keep):
            keep = keep + [ndim - 1]
        merged = []  # list of (shape, gstart, [strides per view], orig_dim or None, is_red)
        for d in keep:
            cur = [shape[d], gs[d], [s[d] for s in strides], d, d in red_dims]
            if merged:
                p = merged[-1]
                can = (p[3] not in iota_dims) and (d not in iota_dims) and (p[4] == cur[4])
                if can and all(p[2][v] == cur[2][v] * cur[0] for v in range(len(strides))):
                    p[0] *= cur[0]
                    p[2] = cur[2]
                    p[3] = None
                    continue
            merged.append(cur)
        if len(merged) > cabi.MAX_DIMS:
            raise cabi.CabiError("fused op iterates over %d non-mergeable dims (max %d)" % (len(merged), cabi.MAX_DIMS))
        fop = cabi.FusedOp()
        fop.abi_version = cabi.ABI_VERSION
        fop.ndim = len(merged)
        iota_remap = {}
        for i, m in enumerate(merged):
            fop.itershape[i] = m[0]
            fop.global_start[i] = m[1]
            if m[3] is not None:
                iota_remap[m[3]] = i
        fop.worker_num = worker_num
        fop.num_workers = num_workers
        fop.n_views = len(bound_views)
        for v, bv in enumerate(bound_views):
            fop.views[v].base = bv[0]
            for i, m in enumerate(merged):
                fop.views[v].stride[i] = m[2][v]
            fop.views[v].dtype = bv[2]
            fop.views[v].flags = 1 if program.view_written.get(v) else 0
            if len(bv) > 3 and bv[3] is not None:
                fop.views[v].alloc_lo, fop.views[v].alloc_hi = bv[3]
        fop.n_scalars = len(program.scalars)
        fop.n_insns = len(program.insns)
        # op list and scalar table are packed once per program and copied in one go
        packed = program.__dict__.get("_packed")
        if packed is None:
            import struct

            ib = b"".join(struct.pack("<12BI", f["op"], f["ctype"], f["a_kind"], f["a_idx"], f["b_kind"], f["b_idx"], f["c_kind"],
                                      f["c_idx"], f["st_reg"], f["st_view"], f["st2"], f["mask_reg"], f["imm"]) for f in program.insns)
            sb = struct.pack("<%dQ" % len(program.scalars), *program.scalars) if program.scalars else b""
            packed = program.__dict__["_packed"] = (ib, sb)
        if packed[0]:
            ctypes.memmove(ctypes.addressof(fop.insns), packed[0], len(packed[0]))
        if packed[1]:
            ctypes.memmove(ctypes.addressof(fop.scalars), packed[1], len(packed[1]))
        if iota_dims:
            for i, f in enumerate(program.insns):
                ins = fop.insns[i]
                for nm in ("a", "b", "c"):
                    if f[nm + "_kind"] == cabi.K_IOTA:
                        od = f[nm + "_idx"]
                        if od not in iota_remap:
                            raise cabi.CabiError("internal: iota over a collapsed dim")
                        setattr(ins, nm + "_idx", iota_remap[od])
        fop.n_regs = program.n_regs
        fop.n_reds = len(program.reds)
        fop.n_axis_red_dims = sum(1 for m in merged if m[4])
        fop.axis_nsplit = axis_nsplit
        if program.reds:
            for s, (rop, rct) in enumerate(program.reds):
                fop.reds[s].op = rop
                fop.reds[s].ctype = rct
                if reds is not None:
                    fop.reds[s].out = reds[s][0]
                    fop.reds[s].out_dtype = reds[s][1]
            if n_axis_red:
                fop.red_scratch = axis_partials
            else:
                fop.red_scratch = self.red_scratch().data_ptr()
        return fop

    def submit(self, fop):
        """Hand one bound op list to the C-ABI on the current stream."""
        be = self.backend or self.be()
        if self.profile_events is not None and be.timing:
            e0, e1 = be.events()
            e0.record()
            be.run(fop, be.stream_handle())
            e1.record()
            self.profile_events.append((e0, e1, fop.n_insns))
        else:
            be.run(fop, be.stream_handle())
        self.launches += 1
        return fop

    # ---- the other kernels of the library, on the current stream.  Counting rule: `launches` counts one per call of a
    # library entry point - a bound op list, a scan, a grouped reduction, a gather, a scatter, a route - whatever number of
    # kernels the call runs; the fold of axis partials (reduce_partials) is not counted.  The methods that return a scratch
    # buffer leave it to the caller to hold (hold()) past the call.
    def reduce_partials(self, out_ptr, in_ptr, n, k, stride_k, code, rop):
        """Fold k partial slices of n elements (stride_k apart) into out (rb200_reduce_partials)."""
        be = self.be()
        be.reduce_partials(out_ptr, in_ptr, n, k, stride_k, code, rop, be.stream_handle())

    def cumulative(self, src_ptr, dst_ptr, code, n_outer, length, n_inner, redop, carry_in=None, totals_out=None):
        """Inclusive scan of one local block through the C-ABI (rb200_cumulative); returns the scratch buffer (or None)."""
        scratch = self.be().cumulative(src_ptr, dst_ptr, code, n_outer, length, n_inner, redop, carry_in, totals_out)
        self.launches += 1
        return scratch

    def group_reduce(self, view, src_code, axis, table, op, center, out):
        """Grouped reduction of one local view along `axis` through the C-ABI (rb200_group_reduce): out (device address,
        accumulator class) receives op over the members of every group (table: a cabi.GroupTable).  Returns the scratch
        buffer (or None)."""
        scratch = self.be().group_reduce(view, src_code, axis, table, op, center, out)
        self.launches += 1
        return scratch

    def arg_reduce(self, view, src_code, axis, op, origin, gstride, out_idx, out_key):
        """First-occurrence index reduction of one local view through the C-ABI (rb200_arg_reduce): over every axis
        (axis = cabi.ARG_ALL_AXES) or along one, writing global indices and order keys to the device addresses out_idx
        and out_key; origin / gstride place the view in the global array.  Returns the scratch buffer (or None)."""
        scratch = self.be().arg_reduce(view, src_code, axis, op, origin, gstride, out_idx, out_key)
        self.launches += 1
        return scratch

    def compact_count(self, cond, cond_code, run_len, counts):
        """Selected elements per chunk of one local condition view cut into runs of run_len C-order positions
        (rb200_compact_count); counts: device address of n_runs * chunks-per-run int64."""
        self.be().compact_count(cond, cond_code, run_len, counts)
        self.launches += 1

    def compact(self, cond, cond_code, run_len, counts, incl, run_base, form, values, origin, gstride, outs):
        """The payload (cabi.COMPACT_VALUES / FLAT / COORDS) of every selected element of one local condition view, in C
        order from run_base[r] + incl[q] - counts[q] for chunk q of run r (rb200_compact); outs: device addresses."""
        self.be().compact(cond, cond_code, run_len, counts, incl, run_base, form, values, origin, gstride, outs)
        self.launches += 1

    def histogram(self, view, src_code, wview, w_code, table, out, bad):
        """This rank's B int64 counts (wview None) or float64 weight sums of one local view into out (device address),
        binned by a cabi.BinTable (rb200_histogram); bad (device uint64) counts the elements no bin may take."""
        keep = self.be().histogram(view, src_code, wview, w_code, table, out, bad)
        self.launches += 1
        return keep

    def bin_search(self, view, src_code, sorted_ptr, n_sorted, sorted_code, side, out):
        """NumPy's searchsorted of every element of one local view in a sorted device table, one int64 per element into
        out in the view's C order (rb200_bin_search)."""
        self.be().bin_search(view, src_code, sorted_ptr, n_sorted, sorted_code, side, out)
        self.launches += 1

    def select_count(self, view, src_code, seg_len, state, pass_, mode):
        """One count pass of the radix select over one local view (or the candidate keys of mode SELECT_CAND) into the
        device counts of a cabi.SelectState (rb200_select_count)."""
        self.be().select_count(view, src_code, seg_len, state, pass_, mode)
        self.launches += 1

    def select_choose(self, view, src_code, seg_len, state, pass_):
        """Every target's bucket of one pass, from the (summed) counts, on the device (rb200_select_choose)."""
        self.be().select_choose(view, src_code, seg_len, state, pass_)
        self.launches += 1

    def select_rows(self, view, src_code, seg_len, targets, rank_table, skip_nan, keys, nans):
        """Every target's key of every segment of one local view, one CTA per segment in shared memory
        (rb200_select_rows)."""
        self.be().select_rows(view, src_code, seg_len, targets, rank_table, skip_nan, keys, nans)
        self.launches += 1

    def gather(self, view, lin, n, out, bad):
        """out[i] = view[lin[i]] for n entries (rb200_gather; view: a cabi.IndexView); bad counts the out-of-range ones."""
        self.be().gather(view, lin, n, out, bad)
        self.launches += 1

    def scatter(self, view, lin, n, values, bad):
        """view[lin[i]] = values[i] for n entries (rb200_scatter); bad counts the out-of-range ones."""
        self.be().scatter(view, lin, n, values, bad)
        self.launches += 1

    def route(self, table, lin, n, offsets, slots, counts, bad):
        """Group n requests by owning rank (rb200_route; table: a cabi.RouteTable); returns the scratch buffer (or None)."""
        scratch = self.be().route(table, lin, n, offsets, slots, counts, bad)
        self.launches += 1
        return scratch

    def synchronize(self):
        if self.backend is not None:
            self.backend.synchronize()


def fill_template(template, views, red_outs=None, red_scratch=None):
    """A copy of the bytes of a bound rb200_fused_op with its addresses filled in.  views: (base, (alloc_lo, alloc_hi) or
    None) per view; red_outs: the output address of every reduction slot, None keeping the template's; red_scratch: None
    keeps the template's."""
    fop = cabi.FusedOp.from_buffer_copy(template)
    fv = fop.views
    for v, (base, bounds) in enumerate(views):
        one = fv[v]
        one.base = base
        if bounds is not None:
            one.alloc_lo, one.alloc_hi = bounds
    if red_outs:
        for sl, out in enumerate(red_outs):
            if out is not None:
                fop.reds[sl].out = out
    if red_scratch is not None:
        fop.red_scratch = red_scratch
    return fop


_launch_cache = {}
# RB200_VERIFY_PLAN_CACHE=1: every hit of the launch memo (here) and of the flush memo (flush.run_deferred_ops) is
# checked against planning the same thing again
_VERIFY_PLAN_CACHE = bool(int(os.environ.get("RB200_VERIFY_PLAN_CACHE", "0")))

RT = Runtime()
