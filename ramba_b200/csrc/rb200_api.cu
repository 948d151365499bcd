// rb200_api.cu — the C-ABI declared in include/ramba_b200.h (host side) and small helper kernels.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <string>

#include "rb200_launch.h"
#include "rb200_plan.h"
#include "rb200_argred.h"
#include "rb200_compact.h"
#include "rb200_hist.h"
#include "rb200_select.h"
#include "rb200_group.h"
#include "rb200_index.h"
#include "rb200_rng.h"
#include "rb200_stream.h"
#include "rb200_tile.h"

namespace rb200 {
__global__ void fill_u64_kernel(u64* p, long long n, u64 bits) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = bits;
}

// stage 2 helper: out[j] = reduce_k part[k*stride_k + j]
template <class T> __global__ void reduce_partials_kernel(T* out, const T* part, long long n, long long k, long long stride_k, int op) {
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x) {
    T v = part[j];
    for (long long q = 1; q < k; ++q) v = red_combine<T>(op, v, part[q * stride_k + j]);
    out[j] = v;
  }
}

}  // namespace rb200

// =============================================================================================
// host side: C-ABI
// =============================================================================================
using namespace rb200;

static thread_local std::string g_last_error;
static std::atomic<long long> g_launches{0};

static int fail(const std::string& msg) {
  g_last_error = msg;
  return 1;
}
static int fail_cuda(const char* what, cudaError_t e) {
  g_last_error = std::string(what) + ": " + cudaGetErrorString(e);
  return 2;
}

static int dtype_size(int dt) {
  switch (dt) {
    case RB200_F64:
    case RB200_I64: return 8;
    case RB200_F32:
    case RB200_I32:
    case RB200_U32: return 4;
    case RB200_I16:
    case RB200_U16: return 2;
    case RB200_BOOL:
    case RB200_U8:
    case RB200_I8: return 1;
    default: return 0;
  }
}

static std::atomic<int> g_sm_count{0};
static int sm_count() {
  const int cached = g_sm_count.load();
  if (cached > 0) return cached;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
  g_sm_count.store(n);
  return n;
}

// the device's multiprocessor count, or the error of every entry point that needs a device
static int need_device(int* sms) {
  *sms = sm_count();
  return *sms > 0 ? 0 : fail("no usable CUDA device (libramba_b200 has no CPU path)");
}

// ---- debugging aids (A/B measurements, bisecting a parity failure), read once: each takes a kernel family, the TMA
// loader, the row tiling or the lean kernel's grid of one CTA per tile out of the selection, in the launch and in
// rb200_describe_plan alike
struct KillSwitches {
  bool no_tile, no_stream, no_mapred, no_terms, no_tma, no_row_mode, no_rng, no_lean, no_cta_per_tile;
};
static const KillSwitches& kill_switches() {
  static const KillSwitches k = {getenv("RB200_NO_TILE_KERNEL") != nullptr,   getenv("RB200_NO_STREAM_KERNEL") != nullptr,
                                 getenv("RB200_NO_MAPRED_KERNEL") != nullptr, getenv("RB200_NO_TERMS_KERNEL") != nullptr,
                                 getenv("RB200_NO_TMA") != nullptr,           getenv("RB200_NO_ROW_MODE") != nullptr,
                                 getenv("RB200_NO_RNG") != nullptr,           getenv("RB200_NO_LEAN_INTERP") != nullptr,
                                 getenv("RB200_NO_CTA_PER_TILE") != nullptr};
  return k;
}

// Every rejection of an op list, before any device query.  0: valid (*empty: an empty range, nothing to run), else the
// status of fail().
static int validate(const rb200_fused_op* op, bool* empty) {
  if (!op) return fail("null fused op");
  if (op->abi_version != RB200_ABI_VERSION) return fail("ABI version mismatch between caller and libramba_b200");
  if (op->ndim < 1 || op->ndim > RB200_MAX_DIMS) return fail("ndim out of range");
  if (op->n_views < 0 || op->n_views > RB200_MAX_VIEWS) return fail("too many views");
  if (op->n_scalars < 0 || op->n_scalars > RB200_MAX_SCALARS) return fail("too many scalars");
  if (op->n_insns < 0 || op->n_insns > RB200_MAX_INSNS) return fail("too many instructions");
  if (op->n_regs < 0 || op->n_regs > RB200_MAX_REGS) return fail("too many spill registers");
  if (op->n_reds < 0 || op->n_reds > RB200_MAX_REDS) return fail("too many reductions");
  long long total = 1;
  for (int d = 0; d < op->ndim; ++d) {
    if (op->itershape[d] < 0) return fail("negative itershape");
    if (op->ndim > 1 && op->itershape[d] >= (1ll << 31)) return fail("N-d iteration dims must be < 2^31");
    total *= op->itershape[d];
  }
  *empty = total == 0 || op->n_insns == 0;
  if (*empty) return 0;

  for (int i = 0; i < op->n_insns; ++i) {
    const rb200_insn& I = op->insns[i];
    if (I.op >= RB200_NUM_OPS) return fail("bad opcode");
    if (I.ctype > RB200_T_I64) return fail("bad compute class");
    const uint8_t kinds[3] = {I.a_kind, I.b_kind, I.c_kind};
    const uint8_t idxs[3] = {I.a_idx, I.b_idx, I.c_idx};
    for (int q = 0; q < 3; ++q) {
      if (!value_slot(I, q)) continue;  // RED's slot and SINCOS's store target: checked below
      switch (kinds[q]) {
        case RB200_K_NONE:
        case RB200_K_ACC: break;
        case RB200_K_REG: if (idxs[q] >= op->n_regs) return fail("register index out of range"); break;
        case RB200_K_VIEW: if (idxs[q] >= op->n_views) return fail("view index out of range"); break;
        case RB200_K_SCAL: if (idxs[q] >= op->n_scalars) return fail("scalar index out of range"); break;
        case RB200_K_IOTA: if (idxs[q] >= op->ndim) return fail("iota dim out of range"); break;
        default: return fail("bad operand kind");
      }
    }
    if (I.op == RB200_OP_SINCOS && I.c_kind == RB200_K_VIEW && I.c_idx >= op->n_views) return fail("view index out of range");
    if (I.st_reg != RB200_NOSTORE && I.st_reg >= op->n_regs) return fail("st_reg out of range");
    if (I.st_view != RB200_NOSTORE && I.st_view >= op->n_views) return fail("st_view out of range");
    if (I.mask_reg != RB200_NOSTORE && I.mask_reg >= op->n_regs) return fail("mask_reg out of range");
    if (I.op == RB200_OP_SINCOS && I.st2 >= op->n_regs) return fail("sincos st2 out of range");
    if (I.op == RB200_OP_RED && I.b_idx >= op->n_reds) return fail("reduction slot out of range");
    if (I.op == RB200_OP_PHILOX) {
      if (I.imm > RB200_PHILOX_INTEGER) return fail("philox: bad output form");
      const int cls = I.imm == RB200_PHILOX_UNIFORM32 ? RB200_T_F32 : I.imm == RB200_PHILOX_INTEGER ? RB200_T_I64 : RB200_T_F64;
      if (I.ctype != cls) return fail("philox: compute class does not match the output form");
      if (I.a_kind != RB200_K_IOTA && I.a_kind != RB200_K_ACC && I.a_kind != RB200_K_REG) return fail("philox: the index must be an index, the accumulator or a register");
      if (I.b_kind != RB200_K_SCAL) return fail("philox: the key must be a scalar");
      if (I.imm == RB200_PHILOX_INTEGER) {
        if (I.c_kind != RB200_K_SCAL) return fail("philox: the integer form needs a scalar bound");
        if ((long long)op->scalars[I.c_idx] <= 0) return fail("philox: the bound must be positive");
      }
    }
  }
  for (int i = 0; i < op->n_views; ++i) {
    if (dtype_size(op->views[i].dtype) == 0) return fail("bad view dtype");
    if (!op->views[i].base) return fail("null view base pointer");
  }
  if (op->n_axis_red_dims != 0) {
    // axis mode: the first n_axis_red_dims dims are the reduced ones (host permutes)
    if (op->n_axis_red_dims >= op->ndim) return fail("axis reduction needs at least one kept dim");
    if (op->n_reds < 1) return fail("axis reduction without reduction slots");
    if (!op->red_scratch) return fail("axis reduction needs a partial buffer");
  } else if (op->n_reds > 0) {
    if (!op->red_scratch) return fail("global reduction needs red_scratch");
    for (int s = 0; s < op->n_reds; ++s) {
      if (!op->reds[s].out) return fail("null reduction output");
      if (dtype_size(op->reds[s].out_dtype) == 0) return fail("bad reduction output dtype");
      if (op->reds[s].ctype != RB200_T_F64 && op->reds[s].ctype != RB200_T_I64) return fail("reduction class must be F64 or I64");
    }
  }
  return 0;
}

enum PlanForm { FORM_NONE, FORM_TILE, FORM_STREAM, FORM_RNG, FORM_INTERP };

// Which kernel runs one op list, and everything its launch needs.  One per call: nothing is shared between calls.
struct Plan {
  PlanForm form;
  TilePlan tile;      // FORM_TILE
  StreamPlan stream;  // FORM_STREAM
  RngPlan rng;        // FORM_RNG
  InterpPlan interp;  // FORM_INTERP
  // axis reductions: the kernel writes splits [0, n_written) of n_split; launch() fills the rest with the identity
  int n_split, n_written;
  long long kept;
  u64* partials;
  u64 identity;
};

static unsigned long long host_red_identity_bits(int op, int ctype) {
  if (ctype == RB200_T_F64) {
    double d = (op == RB200_RED_ADD) ? 0.0 : (op == RB200_RED_MUL) ? 1.0 : (op == RB200_RED_MIN) ? INFINITY : -INFINITY;
    unsigned long long b;
    memcpy(&b, &d, 8);
    return b;
  }
  long long i = (op == RB200_RED_ADD) ? 0ll : (op == RB200_RED_MUL) ? 1ll : (op == RB200_RED_MIN) ? 0x7fffffffffffffffll : (long long)0x8000000000000000ull;
  return (unsigned long long)i;
}

// The kernel choice for a valid, non-empty op list on a device with `sms` multiprocessors.  The only decisions left to
// the launch are the driver's: encoding a TMA tensor map (the cooperative loader when that fails).
static void make_plan(const rb200_fused_op* op, int sms, Plan& pl) {
  const KillSwitches& ks = kill_switches();
  pl.form = FORM_NONE;
  pl.n_split = pl.n_written = 0;
  // ---- a plain random draw (rb200_rng.cu): only op lists with a PHILOX instruction qualify
  if (!ks.no_rng && plan_rng(op, sms, pl.rng)) {
    pl.form = FORM_RNG;
    return;
  }
  // ---- specialised kernels first: float-arithmetic op lists over 2-D / 3-D boxes (shifted-view stencils with the
  // halo tile staged in shared memory by TMA, and N-d elementwise maps) run on the lean machine of rb200_tile.cu
  if (!ks.no_tile && plan_stencil_tile(op, sms, !ks.no_terms, !ks.no_tma, pl.tile)) {
    pl.form = FORM_TILE;
    return;
  }
  if (op->n_axis_red_dims != 0) {
    const AxisBox box = axis_box(op);
    pl.n_split = box.n_split;
    pl.kept = box.kept;
    pl.partials = (u64*)op->red_scratch;
    pl.identity = host_red_identity_bits(op->reds[0].op, op->reds[0].ctype);
  }
  // float-arithmetic op lists over a contiguous 1-D space (incl. global reductions), and the column form of an axis
  // reduction: the streaming kernel
  if ((op->ndim == 1 || op->n_axis_red_dims != 0) && !ks.no_stream && plan_stream(op, sms, pl.n_split, !ks.no_terms, !ks.no_mapred, pl.stream)) {
    pl.form = FORM_STREAM;
    pl.n_written = pl.stream.eff;
    return;
  }
  // ---- the general interpreter
  plan_interp(op, sms, !ks.no_row_mode, !ks.no_lean, !ks.no_cta_per_tile, pl.interp);
  pl.form = FORM_INTERP;
  pl.n_written = pl.interp.n_written;
}

// what a failed launch of the plan's kernel was, for rb200_last_error
static std::string launch_failure(const Plan& pl) {
  const InterpPlan& I = pl.interp;
  char buf[256];
  switch (pl.form) {
    case FORM_TILE: {
      const TilePlan& T = pl.tile;
      snprintf(buf, sizeof(buf), "stencil_tile_kernel launch (blocks=%lld smem=%zu group=%d tma=%d)", T.blocks, T.smem, T.P.has_group, T.P.use_tma);
    } break;
    case FORM_STREAM: {
      const StreamPlan& T = pl.stream;
      snprintf(buf, sizeof(buf), "stream kernel%s launch (blocks=%lld smem=%zu staged=%d depth=%d terms=%d)", T.P.mode == 1 ? " (columns)" : "", T.blocks,
               T.smem, T.P.n_staged, T.P.depth, T.P.n_terms);
    } break;
    case FORM_RNG: snprintf(buf, sizeof(buf), "rng_fill_kernel launch (blocks=%lld)", pl.rng.blocks); break;
    default:
      if (I.form == INTERP_AXIS_AS_1D) return "vm_elementwise_kernel (axis-as-1-D) launch";
      if (I.form == INTERP_AXIS_REDUCE) return "vm_axis_reduce_kernel launch";
      snprintf(buf, sizeof(buf), "vm_elementwise_kernel%s launch (ndim=%d blocks=%lld smem=%zu n_regs=%d n_pf=%d n_insns=%d)", I.lean ? " (lean)" : "", I.k.ndim,
               I.blocks, I.smem, I.k.n_regs, I.k.n_pf, I.k.n_insns);
  }
  return buf;
}

// Launches the plan's kernel and, for an axis reduction whose kernel writes fewer splits than requested, fills the rest
// with the identity.  No choices are made here.
static int launch(Plan& pl, cudaStream_t stream) {
  const InterpPlan& I = pl.interp;
  const KParams& P = I.k;
  const unsigned blocks = (unsigned)I.blocks;
  cudaError_t e = cudaSuccess;
  switch (pl.form) {
    case FORM_NONE: return 0;
    case FORM_TILE: e = launch_stencil_tile(pl.tile, stream); break;
    case FORM_STREAM: e = launch_stream(pl.stream, stream); break;
    case FORM_RNG: e = launch_rng(pl.rng, stream); break;
    case FORM_INTERP:
      if (I.form == INTERP_AXIS_AS_1D) e = launch_vm_elementwise_ax1d(P, blocks, I.smem, stream);
      else if (I.form == INTERP_AXIS_REDUCE) e = launch_vm_axis_reduce(P, blocks, I.smem, stream);
      else if (P.ndim == 1) e = I.lean ? launch_vm_elementwise_lean(P, blocks, I.smem, stream) : launch_vm_elementwise_nd1(P, blocks, I.smem, stream);
      else if (P.ndim == 2) e = launch_vm_elementwise_nd2(P, blocks, I.smem, stream);
      else if (P.ndim == 3) e = launch_vm_elementwise_nd3(P, blocks, I.smem, stream);
      else e = launch_vm_elementwise_nd5(P, blocks, I.smem, stream);
      break;
  }
  if (e != cudaSuccess) return fail_cuda(launch_failure(pl).c_str(), e);
  g_launches.fetch_add(1);
  if (pl.n_written < pl.n_split) {
    const long long n_fill = (long long)(pl.n_split - pl.n_written) * pl.kept;
    fill_u64_kernel<<<(unsigned)((n_fill + 255) / 256 > 1184 ? 1184 : (n_fill + 255) / 256), 256, 0, stream>>>(pl.partials + (long long)pl.n_written * pl.kept,
                                                                                                               n_fill, pl.identity);
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda("fill_u64_kernel launch", e);
    g_launches.fetch_add(1);
  }
  return 0;
}

static std::string describe(const rb200_fused_op* op, const Plan& pl) {
  if (pl.form == FORM_TILE) return describe_stencil_tile(pl.tile);
  if (pl.form == FORM_STREAM) return describe_stream(pl.stream);
  if (pl.form == FORM_RNG) return describe_rng(pl.rng);
  if (pl.form == FORM_INTERP) return describe_interp(op, pl.interp);
  return "kernel=none";
}

// ---- integer-array indexing: argument checks (before any device query, so that they hold on a machine without a GPU)
static int check_index_view(const rb200_index_view* v, const char* who) {
  const std::string w(who);
  if (!v) return fail(w + ": null view");
  if (v->elem_bytes != 1 && v->elem_bytes != 2 && v->elem_bytes != 4 && v->elem_bytes != 8) return fail(w + ": elem_bytes must be 1, 2, 4 or 8");
  if (v->ndim < 1 || v->ndim > RB200_MAX_DIMS) return fail(w + ": ndim out of range");
  long long size = 1, lo = 0, hi = 0;  // element offsets of the first and last reachable element
  for (int d = 0; d < v->ndim; ++d) {
    if (v->shape[d] < 0) return fail(w + ": negative shape");
    size *= v->shape[d];
    const long long reach = (v->shape[d] > 0 ? v->shape[d] - 1 : 0) * v->stride[d];
    if (reach < 0) lo += reach;
    else hi += reach;
  }
  if (size == 0) return 0;
  if (!v->base) return fail(w + ": null view base pointer");
  if (v->alloc_lo && v->alloc_hi) {
    const char* b = (const char*)v->base;
    if (b + lo * v->elem_bytes < (const char*)v->alloc_lo || b + (hi + 1) * v->elem_bytes > (const char*)v->alloc_hi)
      return fail(w + ": view outside its allocation");
  }
  return 0;
}

static int check_route_table(const rb200_route_table* t, RouteParams* R) {
  if (!t) return fail("route: null table");
  if (t->ndim < 1 || t->ndim > RB200_MAX_DIMS) return fail("route: ndim out of range");
  if (t->n_ranks < 1 || t->n_ranks > RB200_MAX_ROUTE_RANKS) return fail("route: too many ranks (or none)");
  if (!t->cuts || !t->cell_owner || !t->cell_offset || !t->cell_stride) return fail("route: null table array");
  R->ndim = t->ndim;
  R->n_ranks = t->n_ranks;
  R->size = 1;
  long long n_cells = 1;
  int n_cuts = 0;
  for (int d = 0; d < t->ndim; ++d) {
    if (t->shape[d] < 0) return fail("route: negative shape");
    if (t->n_cells[d] < 1) return fail("route: not a grid (no cells along a dim)");
    R->shape[d] = t->shape[d];
    R->size *= t->shape[d];
    n_cells *= t->n_cells[d];
    R->n_cells[d] = t->n_cells[d];
    R->cut_start[d] = n_cuts;
    const int first = t->cut_start[d], m = t->n_cells[d] + 1;
    if (first < 0 || n_cuts + m > RB200_MAX_ROUTE_CUTS) return fail("route: too many cut points");
    if (n_cells > RB200_MAX_ROUTE_CELLS) return fail("route: too many cells");
    for (int j = 0; j < m; ++j) R->cuts[n_cuts + j] = t->cuts[first + j];
    if (R->cuts[n_cuts] != 0 || R->cuts[n_cuts + m - 1] != t->shape[d]) return fail("route: not a grid (cuts must run from 0 to the extent)");
    for (int j = 1; j < m; ++j)
      if (R->cuts[n_cuts + j] <= R->cuts[n_cuts + j - 1] && t->shape[d] > 0) return fail("route: not a grid (cuts must ascend)");
    n_cuts += m;
  }
  for (long long c = 0; c < n_cells; ++c) {
    if (t->cell_owner[c] < 0 || t->cell_owner[c] >= t->n_ranks) return fail("route: cell owner out of range");
    R->owner[c] = t->cell_owner[c];
    R->offset[c] = t->cell_offset[c];
    for (int d = 0; d < t->ndim; ++d) R->stride[c * t->ndim + d] = t->cell_stride[c * t->ndim + d];
  }
  return 0;
}

// ---- grouped reduction: argument checks (before any device query) and the plan
static int check_group_args(const rb200_index_view* src, int axis, int n_groups, GroupPlan* P) {
  if (const int rc = check_index_view(src, "group_reduce")) return rc;
  if (axis < 0 || axis >= src->ndim) return fail("group_reduce: axis out of range");
  if (n_groups < 1) return fail("group_reduce: n_groups must be >= 1");
  make_group_plan(*src, axis, n_groups, P);
  if (P->ctas >= (1ll << 31)) return fail("group_reduce: too many outputs for one launch");
  return 0;
}

static thread_local std::string g_group_plan_text;

// ---- index reductions: argument checks (before any device query) and the plan
static int check_arg_args(const rb200_index_view* src, int axis, ArgPlan* P) {
  if (const int rc = check_index_view(src, "arg_reduce")) return rc;
  if (axis != RB200_ARG_ALL_AXES && (axis < 0 || axis >= src->ndim)) return fail("arg_reduce: axis out of range");
  make_arg_plan(*src, axis, P);
  if (P->ctas >= (1ll << 31)) return fail("arg_reduce: too many outputs for one launch");
  return 0;
}

static thread_local std::string g_arg_plan_text;

// ---- stream compaction: argument checks (before any device query) and the plan
static int check_compact_args(const rb200_index_view* cond, long long run_len, CompactPlan* P) {
  if (const int rc = check_index_view(cond, "compact")) return rc;
  make_compact_plan(*cond, run_len, P);
  if (run_len < 1 || P->n % run_len != 0) return fail("compact: run_len must be >= 1 and divide the view's size");
  if (P->ctas >= (1ll << 31)) return fail("compact: too many chunks for one launch");
  return 0;
}

static int check_compact_dtype(const rb200_index_view* cond, int cond_dtype) {
  if (cond_dtype < 0 || cond_dtype >= RB200_NUM_DTYPES) return fail("compact: bad condition dtype");
  if (dtype_size(cond_dtype) != cond->elem_bytes) return fail("compact: elem_bytes does not match the condition dtype");
  return 0;
}

static bool compact_is_float(int dt) { return dt == RB200_F64 || dt == RB200_F32; }

static thread_local std::string g_compact_plan_text;

// ---- binning: argument checks (before any device query) and the plans
static bool bins_src_dtype(int dt) { return dt == RB200_F64 || dt == RB200_F32 || dt == RB200_I64 || dt == RB200_I32; }
static bool bins_float_dtype(int dt) { return dt == RB200_F64 || dt == RB200_F32; }
static bool bins_cmp_dtype(int dt) { return dt == RB200_F64 || dt == RB200_F32 || dt == RB200_I64; }

static int check_bin_table(const rb200_bin_table* T) {
  if (!T) return fail("histogram: null bin table");
  if (T->form != RB200_BINS_UNIFORM && T->form != RB200_BINS_EDGES && T->form != RB200_BINS_INTEGER) return fail("histogram: bad bin table form");
  if (T->n_bins < 1 || T->n_bins > 0x7fffffffll) return fail("histogram: n_bins must be in 1 .. 2^31 - 1");
  if (T->form == RB200_BINS_UNIFORM) {
    if (!bins_float_dtype(T->edge_dtype)) return fail("histogram: uniform edges must be float64 or float32");
    if (!bins_cmp_dtype(T->lo_dtype) || !bins_cmp_dtype(T->hi_dtype)) return fail("histogram: bad bound dtype");
    if (!bins_float_dtype(T->sub_dtype) || !bins_float_dtype(T->div_dtype)) return fail("histogram: bad arithmetic dtype");
    if ((T->edge_dtype == RB200_F64 && T->sub_dtype != RB200_F64) || (T->sub_dtype == RB200_F64 && T->div_dtype != RB200_F64))
      return fail("histogram: arithmetic dtype narrower than the edges");
  } else if (T->form == RB200_BINS_EDGES && !bins_cmp_dtype(T->edge_dtype)) {
    return fail("histogram: bad edge dtype");
  }
  if (T->form != RB200_BINS_INTEGER && !T->edges) return fail("histogram: null edges");
  return 0;
}

static int check_hist_plan(const rb200_index_view* src, bool weighted, const rb200_bin_table* T, HistPlan* P) {
  if (const int rc = check_index_view(src, "histogram")) return rc;
  if (const int rc = check_bin_table(T)) return rc;
  make_hist_plan(*src, weighted, *T, P);
  return 0;
}

static int check_hist_dtypes(const rb200_index_view* src, int src_dtype, const rb200_index_view* weights, int weights_dtype, const rb200_bin_table* T) {
  if (!bins_src_dtype(src_dtype)) return fail("histogram: source dtype must be float64/float32/int64/int32");
  if (dtype_size(src_dtype) != src->elem_bytes) return fail("histogram: elem_bytes does not match the source dtype");
  const bool fl = bins_float_dtype(src_dtype);
  if (fl && T->form == RB200_BINS_INTEGER) return fail("histogram: integer bins need an integer source");
  if (fl && T->form == RB200_BINS_EDGES && T->edge_dtype == RB200_I64) return fail("histogram: integer edges need an integer source");
  if (fl && T->form == RB200_BINS_UNIFORM && (T->lo_dtype == RB200_I64 || T->hi_dtype == RB200_I64))
    return fail("histogram: integer bounds need an integer source");
  if (!weights) return 0;
  if (const int rc = check_index_view(weights, "histogram weights")) return rc;
  if (!bins_src_dtype(weights_dtype)) return fail("histogram: weights dtype must be float64/float32/int64/int32");
  if (dtype_size(weights_dtype) != weights->elem_bytes) return fail("histogram: elem_bytes does not match the weights dtype");
  if (weights->ndim != src->ndim) return fail("histogram: weights and source differ in shape");
  for (int d = 0; d < src->ndim; ++d)
    if (weights->shape[d] != src->shape[d]) return fail("histogram: weights and source differ in shape");
  return 0;
}

static thread_local std::string g_hist_plan_text;

static int check_search_args(const rb200_index_view* src, int src_dtype, const void* sorted, long long n_sorted, int sorted_dtype, int side,
                             SearchPlan* P) {
  if (const int rc = check_index_view(src, "bin_search")) return rc;
  if (!bins_src_dtype(src_dtype)) return fail("bin_search: source dtype must be float64/float32/int64/int32");
  if (dtype_size(src_dtype) != src->elem_bytes) return fail("bin_search: elem_bytes does not match the source dtype");
  if (!bins_cmp_dtype(sorted_dtype)) return fail("bin_search: table dtype must be float64/float32/int64");
  if (sorted_dtype == RB200_I64 && bins_float_dtype(src_dtype)) return fail("bin_search: an integer table needs an integer source");
  if (n_sorted < 0) return fail("bin_search: negative table length");
  if (n_sorted > 0 && !sorted) return fail("bin_search: null table");
  if (side != RB200_SEARCH_LEFT && side != RB200_SEARCH_RIGHT) return fail("bin_search: bad side");
  make_search_plan(*src, n_sorted, sorted_dtype, P);
  P->src_dtype = src_dtype;
  P->side = side;
  return 0;
}

// ---- order statistics: argument checks (before any device query) and the plan
static int check_select_plan(const rb200_index_view* src, int src_dtype, long long seg_len, long long targets, long long segments, SelectPlan* P) {
  if (const int rc = check_index_view(src, "select")) return rc;
  if (!bins_src_dtype(src_dtype)) return fail("select: source dtype must be float64/float32/int64/int32");
  if (dtype_size(src_dtype) != src->elem_bytes) return fail("select: elem_bytes does not match the source dtype");
  long long n = 1;
  for (int d = 0; d < src->ndim; ++d) n *= src->shape[d];
  if (seg_len < 1) return fail("select: seg_len must be at least 1");
  if (n % seg_len != 0) return fail("select: seg_len does not divide the view's size");
  if (targets < 1 || targets > (1ll << 20)) return fail("select: targets must be in 1 .. 2^20");
  if (segments < 0) return fail("select: negative segments");
  if (segments > 0 && n / seg_len > segments) return fail("select: the view holds more segments than the array");
  make_select_plan(*src, src_dtype, seg_len, targets, segments, getenv("RB200_NO_SELECT_ROW") != nullptr, P);
  return 0;
}

static int check_select_state(const SelectPlan& P, const rb200_select_state* st, int pass, const char* who) {
  const std::string w(who);
  if (!st) return fail(w + ": null state");
  if (st->seg_dims < 0 || st->seg_dims > RB200_MAX_DIMS) return fail(w + ": seg_dims out of range");
  if (st->seg_dims == 0 && st->segments != P.S && P.n > 0) return fail(w + ": state segments differ from the view's");
  if (pass < 0 || pass >= P.passes) return fail(w + ": pass out of range");
  if (P.GS > 0 && (!st->rank || !st->key || !st->slot || !st->slot_key || !st->n_slots || !st->counts || !st->nans || !st->matched))
    return fail(w + ": null state buffer");
  return 0;
}

static thread_local std::string g_select_plan_text;

extern "C" {

const char* rb200_last_error(void) { return g_last_error.c_str(); }
int rb200_abi_version(void) { return RB200_ABI_VERSION; }
int64_t rb200_launch_count(void) { return (int64_t)g_launches.load(); }
void rb200_reset_launch_count(void) { g_launches.store(0); }
int rb200_device_sm_count(void) { return sm_count(); }
int64_t rb200_red_scratch_bytes(void) { return (int64_t)kRedScratchBytes; }

int rb200_run_deferred_ops(const rb200_fused_op* op, void* stream_v) {
  bool empty = false;
  if (const int rc = validate(op, &empty)) return rc;
  if (empty) return 0;  // empty range: nothing to do
  // the op list is valid; from here on a device is needed (there is no CPU path)
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  Plan pl;
  make_plan(op, sms, pl);
  return launch(pl, (cudaStream_t)stream_v);
}

int rb200_describe_plan(const rb200_fused_op* op, char* out, int64_t cap) {
  if (!out || cap < 2) return fail("describe_plan: null argument");
  bool empty = false;
  if (const int rc = validate(op, &empty)) return rc;
  Plan pl;
  pl.form = FORM_NONE;
  if (!empty) make_plan(op, 132, pl);  // H100 SXM; the plan does not depend on a device being present
  snprintf(out, (size_t)cap, "%s", describe(op, pl).c_str());
  return 0;
}

int64_t rb200_cumulative_scratch_bytes(int64_t n_outer, int64_t len, int64_t n_inner) {
  if (n_outer < 0 || len < 0 || n_inner < 1) return 256;
  return (int64_t)scan_scratch_bytes(n_outer, len, n_inner);
}

int rb200_cumulative(const void* src, void* dst, int32_t dtype, int64_t n_outer, int64_t len, int64_t n_inner, int32_t redop, const void* carry_in,
                     void* totals_out, void* scratch, void* stream_v) {
  if (n_outer < 0 || len < 0 || n_inner < 1) return fail("cumulative: bad extents");
  if (redop < RB200_RED_ADD || redop > RB200_RED_MAX) return fail("cumulative: bad operation");
  if (dtype != RB200_F64 && dtype != RB200_F32 && dtype != RB200_I64 && dtype != RB200_I32) return fail("cumulative: dtype must be float64/float32/int64/int32");
  if (n_outer == 0 || len == 0) return 0;
  if (!src || !dst || !scratch) return fail("null pointer");
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  bool supported = true;
  const cudaError_t e = launch_scan(src, dst, dtype, n_outer, len, n_inner, redop, carry_in, totals_out, scratch, sms, (cudaStream_t)stream_v, &supported);
  if (!supported) return fail("cumulative: unsupported dtype");
  if (e != cudaSuccess) return fail_cuda("scan kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int rb200_gather(const rb200_index_view* view, const int64_t* lin, int64_t n, void* out, uint64_t* bad, void* stream_v) {
  if (const int rc = check_index_view(view, "gather")) return rc;
  if (n < 0) return fail("gather: negative n");
  if (n == 0) return 0;
  if (!lin || !out || !bad) return fail("gather: null pointer");
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_gather(collapse_index_view(*view), (const long long*)lin, n, out, (unsigned long long*)bad, sms, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("gather kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int rb200_scatter(const rb200_index_view* view, const int64_t* lin, int64_t n, const void* values, uint64_t* bad, void* stream_v) {
  if (const int rc = check_index_view(view, "scatter")) return rc;
  if (n < 0) return fail("scatter: negative n");
  if (n == 0) return 0;
  if (!lin || !values || !bad) return fail("scatter: null pointer");
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e =
      launch_scatter(collapse_index_view(*view), (const long long*)lin, n, values, (unsigned long long*)bad, sms, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("scatter kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int64_t rb200_route_scratch_bytes(int64_t n, int32_t n_ranks) {
  if (n < 0 || n_ranks < 1) return 256;
  return (int64_t)route_scratch_bytes(n, n_ranks);
}

int rb200_route(const rb200_route_table* table, const int64_t* lin, int64_t n, int64_t* offsets, int64_t* slots, int64_t* counts, uint64_t* bad,
                void* scratch, void* stream_v) {
  RouteParams R;
  if (const int rc = check_route_table(table, &R)) return rc;
  if (n < 0) return fail("route: negative n");
  if (!counts || !scratch) return fail("route: null pointer");
  if (n > 0 && (!lin || !offsets || !slots || !bad)) return fail("route: null pointer");
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_route(R, (const long long*)lin, n, (long long*)offsets, (long long*)slots, (long long*)counts,
                                     (unsigned long long*)bad, scratch, sms, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("route kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int64_t rb200_group_reduce_scratch_bytes(const rb200_index_view* src, int32_t axis, int32_t n_groups) {
  GroupPlan P;
  if (check_group_args(src, axis, n_groups, &P)) return -1;
  return (int64_t)P.scratch_bytes;
}

const char* rb200_describe_group_plan(const rb200_index_view* src, int32_t axis, int32_t n_groups) {
  GroupPlan P;
  if (check_group_args(src, axis, n_groups, &P)) return nullptr;
  char buf[240];
  snprintf(buf, sizeof(buf), "kernel=group form=%s chunk=%lld chunks=%d cta_chunks=%d ctas_per_row=%d kept=%lld groups=%d ctas=%lld scratch=%lld",
           group_form_name(P.form), P.C, P.S, P.ncl, P.K, P.nkept, P.G, P.ctas, P.scratch_bytes);
  g_group_plan_text = buf;
  return g_group_plan_text.c_str();
}

int rb200_group_reduce(const rb200_index_view* src, int32_t src_dtype, int32_t axis, const rb200_group_table* groups, int32_t op, const void* center,
                       void* out, void* scratch, void* stream_v) {
  if (op < 0 || op >= RB200_GROUP_NUM_OPS) return fail("group_reduce: bad op");
  if (src_dtype != RB200_F64 && src_dtype != RB200_F32 && src_dtype != RB200_I64 && src_dtype != RB200_I32)
    return fail("group_reduce: source dtype must be float64, float32, int64 or int32");
  if (src && dtype_size(src_dtype) != src->elem_bytes) return fail("group_reduce: elem_bytes does not match the source dtype");
  if (!groups) return fail("group_reduce: null group table");
  GroupPlan P;
  if (const int rc = check_group_args(src, axis, groups->n_groups, &P)) return rc;
  if (groups->len != src->shape[axis]) return fail("group_reduce: table len differs from the extent of the grouped axis");
  if (!groups->offsets || (groups->len > 0 && !groups->members)) return fail("group_reduce: null table array");
  if (op == RB200_GROUP_SQDEV && !center) return fail("group_reduce: SQDEV needs center");
  if (!out) return fail("group_reduce: null out");
  if (P.scratch_bytes && !scratch) return fail("group_reduce: null scratch (this plan splits the axis)");
  if (P.nkept == 0) return 0;
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_group(P, src_dtype, op, (const long long*)groups->offsets, (const long long*)groups->members, (const double*)center, out,
                                     scratch, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("group kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int64_t rb200_arg_reduce_scratch_bytes(const rb200_index_view* src, int32_t axis) {
  ArgPlan P;
  if (check_arg_args(src, axis, &P)) return -1;
  return (int64_t)P.scratch_bytes;
}

const char* rb200_describe_arg_plan(const rb200_index_view* src, int32_t axis) {
  ArgPlan P;
  if (check_arg_args(src, axis, &P)) return nullptr;
  char buf[200];
  snprintf(buf, sizeof(buf), "kernel=argreduce form=%s chunk=%lld split=%d outputs=%lld ctas=%lld scratch=%lld", arg_form_name(P.form), P.C, P.S,
           P.n_out, P.ctas, P.scratch_bytes);
  g_arg_plan_text = buf;
  return g_arg_plan_text.c_str();
}

int rb200_arg_reduce(const rb200_index_view* src, int32_t src_dtype, int32_t axis, int32_t op, const int64_t* origin, const int64_t* gstride,
                     int64_t* out_idx, int64_t* out_key, void* scratch, void* stream_v) {
  if (op < 0 || op >= RB200_ARG_NUM_OPS) return fail("arg_reduce: bad op");
  if (src_dtype != RB200_F64 && src_dtype != RB200_F32 && src_dtype != RB200_I64 && src_dtype != RB200_I32)
    return fail("arg_reduce: source dtype must be float64, float32, int64 or int32");
  if (src && dtype_size(src_dtype) != src->elem_bytes) return fail("arg_reduce: elem_bytes does not match the source dtype");
  ArgPlan P;
  if (const int rc = check_arg_args(src, axis, &P)) return rc;
  if (!origin || !gstride) return fail("arg_reduce: null origin or gstride");
  if (!out_idx || !out_key) return fail("arg_reduce: null out");
  if (P.scratch_bytes && !scratch) return fail("arg_reduce: null scratch (this plan splits the walk)");
  if (P.n_out == 0) return 0;
  bind_arg_coords(*src, axis, (const long long*)origin, (const long long*)gstride, &P);
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_arg(P, src_dtype, op, (long long*)out_idx, (long long*)out_key, scratch, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("arg kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

const char* rb200_describe_compact_plan(const rb200_index_view* cond, int64_t run_len) {
  CompactPlan P;
  if (check_compact_args(cond, run_len, &P)) return nullptr;
  const bool vec = P.cond.nd == 1 && P.cond.stride[0] == 1;
  char buf[256];
  snprintf(buf, sizeof(buf), "kernel=compact runs=%lld run_len=%lld chunk=%d chunks_per_run=%lld runs_per_cta=%lld ctas=%lld load=%s", P.n_runs,
           P.run_len, RB200_COMPACT_CHUNK, P.cpr, P.runs_per_cta, P.ctas, vec ? "vector" : "strided");
  g_compact_plan_text = buf;
  return g_compact_plan_text.c_str();
}

int rb200_compact_count(const rb200_index_view* cond, int32_t cond_dtype, int64_t run_len, int64_t* counts, void* stream_v) {
  CompactPlan P;
  if (const int rc = check_compact_args(cond, run_len, &P)) return rc;
  if (const int rc = check_compact_dtype(cond, cond_dtype)) return rc;
  if (P.n == 0) return 0;
  if (!counts) return fail("compact_count: null counts");
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_compact_count(P, compact_is_float(cond_dtype), (long long*)counts, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("compact count kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int rb200_compact(const rb200_index_view* cond, int32_t cond_dtype, int64_t run_len, const int64_t* counts, const int64_t* incl,
                  const int64_t* run_base, int32_t form, const rb200_index_view* values, const int64_t* origin, const int64_t* gstride,
                  void* const* out, void* stream_v) {
  if (form != RB200_COMPACT_VALUES && form != RB200_COMPACT_FLAT && form != RB200_COMPACT_COORDS) return fail("compact: bad form");
  CompactPlan P;
  if (const int rc = check_compact_args(cond, run_len, &P)) return rc;
  if (const int rc = check_compact_dtype(cond, cond_dtype)) return rc;
  CompactOut O;
  O.form = form;
  O.k = form == RB200_COMPACT_COORDS ? cond->ndim : 1;
  O.g0 = 0;
  if (form == RB200_COMPACT_VALUES) {
    if (const int rc = check_index_view(values, "compact values")) return rc;
    if (values->ndim != cond->ndim) return fail("compact: values and condition differ in shape");
    for (int d = 0; d < cond->ndim; ++d)
      if (values->shape[d] != cond->shape[d]) return fail("compact: values and condition differ in shape");
    O.values = make_compact_view(*values);
  } else {
    if (!origin || (form == RB200_COMPACT_FLAT && !gstride)) return fail("compact: null origin or gstride");
    for (int d = 0; d < cond->ndim; ++d) {
      O.cshape[d] = cond->shape[d];
      O.origin[d] = origin[d];
      O.gstride[d] = form == RB200_COMPACT_FLAT ? gstride[d] : 0;
      O.g0 += O.origin[d] * O.gstride[d];
    }
    if (form == RB200_COMPACT_FLAT) O.k = cond->ndim;
  }
  if (P.n == 0) return 0;
  if (!counts || !incl || !run_base) return fail("compact: null counts, incl or run_base");
  if (!out) return fail("compact: null out");
  const int n_out = form == RB200_COMPACT_COORDS ? cond->ndim : 1;
  for (int i = 0; i < n_out; ++i) {
    if (!out[i]) return fail("compact: null out");
    O.out[i] = out[i];
  }
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_compact(P, compact_is_float(cond_dtype), (const long long*)counts, (const long long*)incl, (const long long*)run_base, O,
                                       (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("compact kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

const char* rb200_describe_hist_plan(const rb200_index_view* src, int32_t weighted, const rb200_bin_table* table) {
  HistPlan P;
  if (check_hist_plan(src, weighted != 0, table, &P)) return nullptr;
  char buf[320];
  snprintf(buf, sizeof(buf),
           "kernel=hist form=%s bins=%lld chunk=%lld ctas=%lld warps=%d shared_bytes=%lld passes=%lld slab=%lld table=%s load=%s scratch=%lld",
           hist_form_name(P.form), P.B, P.chunk, P.ctas, 8, P.shared_bytes, P.passes, P.slab,
           table->form == RB200_BINS_INTEGER ? "none" : P.table_shared ? "shared" : "global", P.vec ? "vector" : "strided", P.scratch_bytes);
  g_hist_plan_text = buf;
  return g_hist_plan_text.c_str();
}

int64_t rb200_histogram_scratch_bytes(const rb200_index_view* src, int32_t weighted, const rb200_bin_table* table) {
  HistPlan P;
  if (check_hist_plan(src, weighted != 0, table, &P)) return -1;
  return P.scratch_bytes;
}

int rb200_histogram(const rb200_index_view* src, int32_t src_dtype, const rb200_index_view* weights, int32_t weights_dtype,
                    const rb200_bin_table* table, void* out, uint64_t* bad, void* scratch, void* stream_v) {
  HistPlan P;
  if (const int rc = check_hist_plan(src, weights != nullptr, table, &P)) return rc;
  if (const int rc = check_hist_dtypes(src, src_dtype, weights, weights_dtype, table)) return rc;
  P.src_dtype = src_dtype;
  P.w_dtype = weights_dtype;
  if (!out) return fail("histogram: null out");
  if (!bad && table->form != RB200_BINS_EDGES) return fail("histogram: null bad counter");
  if (P.n > 0 && P.scratch_bytes > 0 && !scratch) return fail("histogram: null scratch");
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_histogram(P, *table, weights, out, (unsigned long long*)bad, scratch, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("histogram kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int rb200_bin_search(const rb200_index_view* src, int32_t src_dtype, const void* sorted, int64_t n_sorted, int32_t sorted_dtype, int32_t side,
                     int64_t* out, void* stream_v) {
  SearchPlan P;
  if (const int rc = check_search_args(src, src_dtype, sorted, n_sorted, sorted_dtype, side, &P)) return rc;
  if (P.n == 0) return 0;
  if (!out) return fail("bin_search: null out");
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_bin_search(P, sorted, (long long*)out, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("bin search kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

const char* rb200_describe_select_plan(const rb200_index_view* src, int32_t src_dtype, int64_t seg_len, int64_t targets, int64_t segments) {
  SelectPlan P;
  if (check_select_plan(src, src_dtype, seg_len, targets, segments, &P)) return nullptr;
  char buf[320];
  snprintf(buf, sizeof(buf),
           "kernel=select form=%s segments=%lld all_segments=%lld seg_len=%lld targets=%lld digit=%d passes=%d ctas=%lld chunk=%lld rows=%lld groups=%lld "
           "shared_bytes=%lld counts_bytes=%lld scratch_bytes=%lld load=%s",
           select_form_name(P.form), P.S, P.GS, P.L, P.K, P.digit, P.passes, P.ctas, P.chunk, P.rows, P.groups, P.shared_bytes, P.counts_bytes,
           P.cand_cap * 8, P.vec ? "vector" : "strided");
  g_select_plan_text = buf;
  return g_select_plan_text.c_str();
}

int64_t rb200_select_scratch_bytes(const rb200_index_view* src, int32_t src_dtype, int64_t seg_len, int64_t targets, int64_t segments) {
  SelectPlan P;
  if (check_select_plan(src, src_dtype, seg_len, targets, segments, &P)) return -1;
  return P.cand_cap * 8;
}

int rb200_select_count(const rb200_index_view* src, int32_t src_dtype, int64_t seg_len, const rb200_select_state* state, int32_t pass,
                       int32_t mode, void* stream_v) {
  SelectPlan P;
  if (!state) return fail("select_count: null state");
  if (const int rc = check_select_plan(src, src_dtype, seg_len, state->targets, std::max<long long>(state->segments, 1), &P)) return rc;
  if (const int rc = check_select_state(P, state, pass, "select_count")) return rc;
  if (mode != RB200_SELECT_READ && mode != RB200_SELECT_APPEND && mode != RB200_SELECT_CAND) return fail("select_count: bad mode");
  if (mode != RB200_SELECT_READ) {
    if (P.GS != 1) return fail("select_count: candidate compaction needs one segment");
    if (pass == 0) return fail("select_count: candidate compaction needs a chosen prefix (pass >= 1)");
    if (!state->cand || !state->cand_n || state->cand_cap < 1)
      return fail("select_count: bad candidate buffer");
  }
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_select_count(P, *state, pass, mode, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("select count kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int rb200_select_choose(const rb200_index_view* src, int32_t src_dtype, int64_t seg_len, const rb200_select_state* state, int32_t pass,
                        void* stream_v) {
  SelectPlan P;
  if (!state) return fail("select_choose: null state");
  if (const int rc = check_select_plan(src, src_dtype, seg_len, state->targets, std::max<long long>(state->segments, 1), &P)) return rc;
  if (const int rc = check_select_state(P, state, pass, "select_choose")) return rc;
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_select_choose(P, *state, pass, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("select choose kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int rb200_select_rows(const rb200_index_view* src, int32_t src_dtype, int64_t seg_len, int64_t targets, const int64_t* rank_table,
                      int32_t skip_nan, uint64_t* keys, int64_t* nans, void* stream_v) {
  SelectPlan P;
  if (const int rc = check_select_plan(src, src_dtype, seg_len, targets, 0, &P)) return rc;
  if (P.form != SELECT_ROW) return fail("select_rows: the segments do not fit in shared memory (rb200_select_count)");
  if (P.S > 0 && (!rank_table || !keys || !nans)) return fail("select_rows: null rank table, keys or nans");
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  const cudaError_t e = launch_select_rows(P, (const long long*)rank_table, skip_nan != 0, (unsigned long long*)keys, (long long*)nans,
                                           (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("select row kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int rb200_reduce_partials(void* out, const void* partials, int64_t n, int64_t k, int64_t stride_k, int32_t dtype,
                          int32_t redop, void* stream_v) {
  if (!out || !partials) return fail("null pointer");
  if (n <= 0 || k <= 0) return 0;
  int sms;
  if (const int rc = need_device(&sms)) return rc;
  cudaStream_t stream = (cudaStream_t)stream_v;
  long long blocks = (n + 255) / 256;
  if (blocks > sms * 8) blocks = sms * 8;
  if (dtype == RB200_F64)
    reduce_partials_kernel<double><<<(unsigned)blocks, 256, 0, stream>>>((double*)out, (const double*)partials, n, k, stride_k, redop);
  else if (dtype == RB200_I64)
    reduce_partials_kernel<long long><<<(unsigned)blocks, 256, 0, stream>>>((long long*)out, (const long long*)partials, n, k, stride_k, redop);
  else
    return fail("reduce_partials: dtype must be F64 or I64 (accumulator classes)");
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail_cuda("reduce_partials_kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

}  // extern "C"
