// rb200_api.cu — the C-ABI declared in include/ramba_b200.h (host side) and small helper kernels.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <string>

#include "rb200_launch.h"
#include "rb200_handlers.h"
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

constexpr int kRedScratchPartials = 4096;  // max grid size of a launch with global reductions

// static operand kind of an op-list operand for the specialised handlers (-1: needs the generic path);
// staged views are addressed by their prefetch slot (*idx is rewritten)
static int static_kind(const KParams& P, int set, int kind, int* idx, int ctype) {
  switch (kind) {
    case RB200_K_ACC: return S_ACC;
    case RB200_K_REG: return S_REG;
    case RB200_K_SCAL: return S_SCAL;
    case RB200_K_VIEW: {
      const KView& v = P.views[*idx];
      const int own = ctype == RB200_T_F64 ? RB200_F64 : ctype == RB200_T_F32 ? RB200_F32 : RB200_I64;
      if (set == 2) {  // N-d kernels: direct views
        if (v.dtype == own) return S_VIEW;
        if (ctype == RB200_T_F64 && v.dtype == RB200_F32) return S_VIEW32;
        return -1;
      }
      if (v.pf_slot < 0) return -1;
      if (v.dtype == own) {
        *idx = v.pf_slot;
        return S_PFV;
      }
      if (ctype == RB200_T_F64 && v.dtype == RB200_F32) {
        *idx = v.pf_slot;
        return S_PFV32;
      }
      return -1;
    }
    default: return -1;
  }
}

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

static void assign_handlers(KParams& P, const rb200_fused_op* op, int set) {
  for (int i = 0; i < P.n_insns; ++i) {
    rb200_insn I = P.insns[i];
    int h = H_GENERIC;
    int ai = I.a_idx, bi = I.b_idx;
    // CVT fetches its operand in the SOURCE class (imm & 0xff)
    const int ak = static_kind(P, set, I.a_kind, &ai, I.op == RB200_OP_CVT ? (int)(I.imm & 0xff) : (int)I.ctype);
    if (I.op == RB200_OP_ADD || I.op == RB200_OP_SUB || I.op == RB200_OP_MUL) {
      const int bk = static_kind(P, set, I.b_kind, &bi, I.ctype);
      h = handler_bin(set, I.op, I.ctype, ak, bk);
    } else if (I.op == RB200_OP_RED) {
      h = handler_red(set, I.ctype, ak);
    } else if (I.op == RB200_OP_CVT) {
      if ((I.imm >> 8) == 0) h = handler_cvt(set, (int)(I.imm & 0xff), I.ctype, ak);
    } else if (I.op == RB200_OP_POWI) {
      // only x ** 2 with a scalar exponent (Numba int_power gives exactly x*x)
      if (I.b_kind == RB200_K_SCAL && (long long)op->scalars[I.b_idx] == 2) h = handler_un(set, I.op, I.ctype, ak);
    } else if ((I.c_kind == RB200_K_NONE || I.op == RB200_OP_SINCOS) && I.b_kind == RB200_K_NONE) {
      h = handler_un(set, I.op, I.ctype, ak);
    }
    if (h != H_GENERIC) {
      I.a_idx = (uint8_t)ai;
      if (I.op != RB200_OP_RED) I.b_idx = (uint8_t)bi;
      P.insns[i] = I;
    }
    P.handler[i] = (unsigned short)h;
  }
}

// ---- debugging aids (A/B measurements, bisecting a parity failure), read once: each takes a kernel family, the TMA
// loader or the row tiling out of the selection, in the launch and in rb200_describe_plan alike
struct KillSwitches {
  bool no_tile, no_stream, no_mapred, no_terms, no_tma, no_row_mode, no_rng, no_lean;
};
static const KillSwitches& kill_switches() {
  static const KillSwitches k = {getenv("RB200_NO_TILE_KERNEL") != nullptr,   getenv("RB200_NO_STREAM_KERNEL") != nullptr,
                                 getenv("RB200_NO_MAPRED_KERNEL") != nullptr, getenv("RB200_NO_TERMS_KERNEL") != nullptr,
                                 getenv("RB200_NO_TMA") != nullptr,           getenv("RB200_NO_ROW_MODE") != nullptr,
                                 getenv("RB200_NO_RNG") != nullptr,           getenv("RB200_NO_LEAN_INTERP") != nullptr};
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
      if (I.op == RB200_OP_RED && q == 1) continue;     // b_idx is the slot
      if (I.op == RB200_OP_SINCOS && q == 2) {          // c names the view the parked half is stored to
        if (kinds[q] == RB200_K_VIEW && idxs[q] >= op->n_views) return fail("view index out of range");
        continue;
      }
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

enum PlanForm { FORM_NONE, FORM_TILE, FORM_STREAM, FORM_AXIS_AS_1D, FORM_AXIS_REDUCE, FORM_ELEMENTWISE, FORM_RNG };

// Which kernel runs one op list, and everything its launch needs.  One per call: nothing is shared between calls.
struct Plan {
  PlanForm form;
  TilePlan tile;      // FORM_TILE
  StreamPlan stream;  // FORM_STREAM
  RngPlan rng;        // FORM_RNG
  KParams k;          // the general interpreter forms
  bool lean;          // FORM_ELEMENTWISE, 1-D: the lean instantiation (handler ids are lean ids)
  long long blocks;   // the general interpreter forms: grid and dynamic shared memory
  size_t smem;
  // axis reductions: the kernel writes splits [0, n_written) of n_split; launch() fills the rest with the identity
  int n_split, n_written;
  long long kept;
  u64* partials;
  u64 identity;
};

// axis-as-1-D form: [R reduced rows][C kept elements], every view contiguous over the box or broadcast over the rows,
// C a multiple of the 1-D tile, one reduction slot, no index operands: the staged 1-D kernel with V column accumulators
// per thread (rb200_elementwise_ax1d.cu).  false: not of this form, or its shared memory does not fit.
static bool plan_axis_as_1d(const rb200_fused_op* op, int sms, const bool* view_read, size_t reg_bytes, Plan& pl) {
  const KParams& P = pl.k;
  const long long TILE1 = (long long)kThreads * kV1;
  const long long red_len = P.red_len, kept = P.total;
  bool ok = (op->ndim == 2 && P.red_ndim == 1 && op->n_reds == 1 && kept % TILE1 == 0 && kept / TILE1 <= (long long)sms * 2 && red_len >= 2);
  for (int i = 0; i < op->n_insns && ok; ++i) {
    const rb200_insn& I = op->insns[i];
    if (I.a_kind == RB200_K_IOTA || I.b_kind == RB200_K_IOTA || I.c_kind == RB200_K_IOTA) ok = false;
    if (I.st_view != RB200_NOSTORE) ok = false;  // stage 1 of an axis reduction only reads
    if (I.op == RB200_OP_SINCOS && I.c_kind == RB200_K_VIEW) ok = false;  // (the parked-half store is a write too)
  }
  for (int i = 0; i < op->n_views && ok; ++i) {
    const rb200_view& v = op->views[i];
    if (!view_read[i]) continue;
    if (v.stride[1] != 1 || !(v.stride[0] == kept || v.stride[0] == 0)) ok = false;
  }
  if (!ok) return false;
  KParams Q = P;
  const int V1 = kV1;
  Q.ndim = 1;
  Q.total = red_len * kept;
  Q.n_tiles = Q.total / TILE1;
  Q.shape[0] = Q.total;
  Q.gstart[0] = 0;
  Q.wide = 1;
  const int n_chunks = (int)(kept / TILE1);
  long long cap1 = (long long)sms * 2;
  int n_split_eff = (int)(cap1 / n_chunks);
  if (n_split_eff > P.n_split) n_split_eff = P.n_split;
  if ((long long)n_split_eff > red_len) n_split_eff = (int)red_len;
  if (n_split_eff < 1) n_split_eff = 1;
  Q.n_split_chunks = n_chunks;
  Q.n_split = n_split_eff;
  Q.red_len = kept;  // in this mode: elements per row (partials are [split][kept])
  Q.n_pf = 0;
  for (int i = 0; i < op->n_views; ++i) {
    KView& k = Q.views[i];
    const rb200_view& v = op->views[i];
    k.stride[0] = 1;
    k.pf_slot = -1;
    if (!view_read[i]) continue;
    const int dt = v.dtype;
    const bool wide_ok = (dt == RB200_F64 || dt == RB200_F32 || dt == RB200_I64 || dt == RB200_I32);
    if (v.stride[0] == 0) {
      k.pf_slot = -2;  // periodic: broadcast over the rows
    } else if (wide_ok && Q.n_pf < kMaxPf && reg_bytes + (size_t)(Q.n_pf + 1) * 2 * V1 * kThreads * 8 <= 108 * 1024) {
      k.pf_slot = Q.n_pf;
      Q.pf_view[Q.n_pf] = i;
      Q.n_pf++;
    }
  }
  // hoist periodic views into extra spill registers when every use agrees on the compute class
  for (int i = 0; i < op->n_views && Q.n_hoist < kMaxPf; ++i) {
    if (Q.views[i].pf_slot != -2 || Q.n_regs >= RB200_MAX_REGS) continue;
    int cls = -1;
    bool same = true;
    for (int q = 0; q < Q.n_insns; ++q) {
      const rb200_insn& I = Q.insns[q];
      const int use_cls = (I.op == RB200_OP_CVT) ? (int)(I.imm & 0xff) : (int)I.ctype;
      const bool uses = (I.a_kind == RB200_K_VIEW && I.a_idx == i) || (I.b_kind == RB200_K_VIEW && I.b_idx == i && I.op != RB200_OP_RED) ||
                        (I.c_kind == RB200_K_VIEW && I.c_idx == i && I.op != RB200_OP_SINCOS);
      if (!uses) continue;
      if (I.op == RB200_OP_POWI && I.b_kind == RB200_K_VIEW && I.b_idx == i) same = false;  // integer exponent operand
      if (cls < 0) cls = use_cls;
      else if (cls != use_cls) same = false;
    }
    if (cls < 0 || !same) continue;
    const int r = Q.n_regs++;
    Q.hoist_view[Q.n_hoist] = i;
    Q.hoist_reg[Q.n_hoist] = r;
    Q.hoist_cls[Q.n_hoist] = cls;
    Q.n_hoist++;
    for (int q = 0; q < Q.n_insns; ++q) {
      rb200_insn& I = Q.insns[q];
      if (I.a_kind == RB200_K_VIEW && I.a_idx == i) { I.a_kind = RB200_K_REG; I.a_idx = (uint8_t)r; }
      if (I.b_kind == RB200_K_VIEW && I.b_idx == i && I.op != RB200_OP_RED) { I.b_kind = RB200_K_REG; I.b_idx = (uint8_t)r; }
      if (I.c_kind == RB200_K_VIEW && I.c_idx == i && I.op != RB200_OP_SINCOS) { I.c_kind = RB200_K_REG; I.c_idx = (uint8_t)r; }
    }
  }
  const size_t reg_bytes1 = (size_t)(Q.n_regs + 1) * V1 * kThreads * 8;
  Q.bulk = Q.n_pf > 0 ? 1 : 0;
  for (int j = 0; j < Q.n_pf; ++j)
    if ((((uintptr_t)op->views[Q.pf_view[j]].base) & 15u) != 0) Q.bulk = 0;
  Q.n_stages = 2;
  const size_t pf_bytes1 = (size_t)Q.n_pf * Q.n_stages * V1 * kThreads * 8;
  if (reg_bytes1 + pf_bytes1 > 200 * 1024) return false;  // does not fit: the general axis kernel runs it
  assign_handlers(Q, op, 1);
  pl.k = Q;
  pl.form = FORM_AXIS_AS_1D;
  pl.blocks = (long long)n_split_eff * n_chunks;
  pl.smem = reg_bytes1 + pf_bytes1;
  pl.n_written = n_split_eff;
  return true;
}

// The lean 1-D kernel (rb200_elementwise_lean.cu) runs a 1-D op list, already staged and given its set-1 handlers, when
// every instruction has a handler of the lean set, nothing is reduced, every store is unmasked and goes to a contiguous
// view of the result's own dtype, and the staged views move by bulk copies: what the lean kernel leaves out (the generic
// path, reductions, converting / masked / strided stores, the per-thread staging pipeline) is then never needed.
static bool lean_eligible(const KParams& P, const rb200_fused_op* op) {
  if (P.ndim != 1 || op->n_reds != 0 || (P.n_pf > 0 && !P.bulk)) return false;
  for (int i = 0; i < P.n_insns; ++i) {
    const rb200_insn& I = P.insns[i];
    const int h = P.handler[i];
    if (h == H_GENERIC || kLeanOf1[h] == 0) return false;
    if (I.st_view != RB200_NOSTORE && I.mask_reg != RB200_NOSTORE) return false;
    const int own = I.ctype == RB200_T_F64 ? RB200_F64 : RB200_F32;  // the lean set is float64 / float32 only
    const int stored[2] = {I.st_view, (I.op == RB200_OP_SINCOS && I.c_kind == RB200_K_VIEW) ? (int)I.c_idx : RB200_NOSTORE};
    for (const int v : stored)
      if (v != RB200_NOSTORE && (P.views[v].stride[0] != 1 || P.views[v].dtype != own)) return false;
  }
  return true;
}

// The kernel choice for a valid, non-empty op list on a device with `sms` multiprocessors.  The only decisions left to
// the launch are the driver's: encoding a TMA tensor map (the cooperative loader when that fails).
static void make_plan(const rb200_fused_op* op, int sms, Plan& pl) {
  const KillSwitches& ks = kill_switches();
  pl.form = FORM_NONE;
  pl.lean = false;
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
  // float-arithmetic op lists over a contiguous 1-D space (incl. global reductions): the streaming kernel
  if (op->ndim == 1 && op->n_axis_red_dims == 0 && !ks.no_stream &&
      plan_stream(op, sms, kRedScratchPartials, 0, !ks.no_terms, !ks.no_mapred, pl.stream)) {
    pl.form = FORM_STREAM;
    return;
  }

  // ---- the general interpreter
  // the 1-D kernel owns 8 elements per thread, the N-d and axis kernels 4
  const int V = (op->ndim == 1 && op->n_axis_red_dims == 0) ? kV1 : kV;
  const long long TILE = (long long)kThreads * V;
  KParams& P = pl.k;
  memset(&P, 0, sizeof(P));
  P.ndim = op->ndim;
  P.n_insns = op->n_insns;
  P.n_views = op->n_views;
  P.n_regs = op->n_regs;
  P.n_reds = op->n_reds;
  long long total = 1;
  for (int d = 0; d < op->ndim; ++d) {
    P.shape[d] = op->itershape[d];
    P.gstart[d] = op->global_start[d];
    total *= op->itershape[d];
  }
  bool view_read[RB200_MAX_VIEWS] = {false}, view_masked[RB200_MAX_VIEWS] = {false};
  for (int i = 0; i < op->n_insns; ++i) {
    const rb200_insn& I = op->insns[i];
    const uint8_t kinds[3] = {I.a_kind, I.b_kind, I.c_kind};
    const uint8_t idxs[3] = {I.a_idx, I.b_idx, I.c_idx};
    for (int q = 0; q < 3; ++q)
      if (kinds[q] == RB200_K_VIEW && !(I.op == RB200_OP_RED && q == 1) && !(I.op == RB200_OP_SINCOS && q == 2)) view_read[idxs[q]] = true;
    if (I.st_view != RB200_NOSTORE && I.mask_reg != RB200_NOSTORE) view_masked[I.st_view] = true;
    P.insns[i] = I;
  }
  for (int i = 0; i < op->n_scalars; ++i) P.scalars[i] = op->scalars[i];
  for (int i = 0; i < op->n_views; ++i) {
    const rb200_view& v = op->views[i];
    KView& k = P.views[i];
    k.base = (char*)v.base;
    k.dtype = v.dtype;
    k.pf_slot = -1;
    for (int d = 0; d < op->ndim; ++d) k.stride[d] = v.stride[d];
  }
  const size_t reg_bytes = (size_t)(op->n_regs + 1) * V * kThreads * 8;  // + the scratch column of the out-of-line stores

  if (op->n_axis_red_dims != 0) {
    const int nred = op->n_axis_red_dims;
    P.red_ndim = nred;
    long long red_len = 1, kept = 1;
    for (int d = 0; d < nred; ++d) red_len *= P.shape[d];
    for (int d = nred; d < op->ndim; ++d) kept *= P.shape[d];
    int n_split = op->axis_nsplit;
    if (n_split < 1) n_split = 1;
    if ((long long)n_split > red_len) n_split = (int)red_len;
    P.red_len = red_len;
    P.n_split = n_split;
    P.red_split = (red_len + n_split - 1) / n_split;
    P.total = kept;
    P.n_tiles = ((kept + TILE - 1) / TILE) * n_split;
    P.red_partials = (u64*)op->red_scratch;
    for (int s = 0; s < op->n_reds; ++s) {
      P.reds[s].op = op->reds[s].op;
      P.reds[s].ctype = op->reds[s].ctype;
    }
    pl.n_split = n_split;
    pl.kept = kept;
    pl.partials = (u64*)op->red_scratch;
    pl.identity = host_red_identity_bits(op->reds[0].op, op->reds[0].ctype);
    // ---- column form on the streaming kernel of the lean machine (float arithmetic op lists)
    if (!ks.no_stream && plan_stream(op, sms, kRedScratchPartials, n_split, !ks.no_terms, !ks.no_mapred, pl.stream)) {
      pl.form = FORM_STREAM;
      pl.n_written = pl.stream.eff;
      return;
    }
    if (plan_axis_as_1d(op, sms, view_read, reg_bytes, pl)) return;
    long long blocks = P.n_tiles;
    long long cap = (long long)sms * 4;
    if (blocks > cap) blocks = cap;
    pl.form = FORM_AXIS_REDUCE;
    pl.blocks = blocks;
    pl.smem = reg_bytes;
    pl.n_written = n_split;
    return;
  }

  P.total = total;
  P.n_tiles = (total + TILE - 1) / TILE;
  P.row_chunks = 0;
  if (op->ndim > 1) {
    // row mode: tiles are cut along the innermost dim only, so the outer indices are decoded once per
    // tile instead of once per element (no per-element divisions); used when rows fill their tiles well
    const long long inner = op->itershape[op->ndim - 1];
    const long long chunks = (inner + TILE - 1) / TILE;
    if (!ks.no_row_mode && inner * 5 >= chunks * TILE * 4 && chunks < (1ll << 30)) {
      P.row_chunks = (int)chunks;
      P.n_tiles = (total / inner) * chunks;
    }
  }
  P.wide = (total >= (1ll << 31)) ? 1 : 0;
  // stage read-only 4/8-byte input views of 1-D ops one tile ahead through shared memory
  size_t pf_bytes = 0;
  if (op->ndim == 1) {
    for (int i = 0; i < op->n_views && P.n_pf < kMaxPf; ++i) {
      const int dt = op->views[i].dtype;
      const bool wide_ok = (dt == RB200_F64 || dt == RB200_F32 || dt == RB200_I64 || dt == RB200_I32);
      if (view_read[i] && !view_masked[i] && wide_ok && reg_bytes + (size_t)(P.n_pf + 1) * 2 * V * kThreads * 8 <= 108 * 1024) {
        P.views[i].pf_slot = P.n_pf;
        P.pf_view[P.n_pf] = i;
        P.n_pf++;
      }
    }
    P.n_stages = 2;  // two-stage ring: the next tile is in flight while the current one is interpreted
    pf_bytes = (size_t)P.n_pf * P.n_stages * V * kThreads * 8;
    // whole-tile bulk copies need contiguous, 16-byte aligned sources
    P.bulk = P.n_pf > 0 ? 1 : 0;
    for (int j = 0; j < P.n_pf; ++j) {
      const rb200_view& v = op->views[P.pf_view[j]];
      if (v.stride[0] != 1 || (((uintptr_t)v.base) & 15u) != 0) P.bulk = 0;
    }
  }
  size_t ocls_bytes = 0;
  if (op->ndim > 1) {
    // offset classes: views with identical stride vectors (the shifted views of a stencil, operands
    // of the same shape) share their per-tile element offsets
    for (int i = 0; i < op->n_views; ++i) {
      int c = -1;
      for (int q = 0; q < P.n_ocls && c < 0; ++q) {
        bool same = true;
        for (int d = 0; d < op->ndim; ++d)
          if (op->views[P.ocls_view[q]].stride[d] != op->views[i].stride[d]) same = false;
        if (same) c = q;
      }
      if (c < 0 && P.n_ocls < kMaxOcls) {
        c = P.n_ocls;
        P.ocls_view[P.n_ocls++] = i;
      }
      P.views[i].pf_slot = c;
    }
    ocls_bytes = (size_t)P.n_ocls * V * kThreads * 8;
  }
  assign_handlers(P, op, op->ndim == 1 ? 1 : 2);
  if (!ks.no_lean && lean_eligible(P, op)) {
    pl.lean = true;
    for (int i = 0; i < P.n_insns; ++i) P.handler[i] = kLeanOf1[P.handler[i]];
  }
  // (the lean kernel's stores never go through the scratch column behind the register file)
  const size_t smem = (pl.lean ? reg_bytes - (size_t)V * kThreads * 8 : reg_bytes) + pf_bytes + ocls_bytes;
  if (op->n_reds > 0) {
    P.red_counter = (unsigned int*)op->red_scratch;
    P.red_partials = (u64*)((char*)op->red_scratch + 256);
    for (int s = 0; s < op->n_reds; ++s) {
      P.reds[s].op = op->reds[s].op;
      P.reds[s].ctype = op->reds[s].ctype;
      P.reds[s].out = op->reds[s].out;
      P.reds[s].out_dtype = op->reds[s].out_dtype;
    }
  }
  // persistent-style grid: SM count x resident CTAs per SM (smem / register limited), capped by
  // the number of tiles; every CTA walks tiles b, b+grid, ...
  int per_sm = (V == 4 && op->ndim == 1) ? 3 : 2;
  if (smem > 0) {
    int by_smem = (int)((220 * 1024) / (smem + 1024));
    if (by_smem < 1) by_smem = 1;
    if (per_sm > by_smem) per_sm = by_smem;
  }
  long long blocks = P.n_tiles;
  long long cap = (long long)sms * per_sm;
  if (op->n_reds > 0 && cap > kRedScratchPartials) cap = kRedScratchPartials;
  if (blocks > cap) blocks = cap;
  pl.form = FORM_ELEMENTWISE;
  pl.blocks = blocks;
  pl.smem = smem;
}

// what a failed launch of the plan's kernel was, for rb200_last_error
static std::string launch_failure(const Plan& pl) {
  const KParams& P = pl.k;
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
    case FORM_AXIS_AS_1D: return "vm_elementwise_kernel (axis-as-1-D) launch";
    case FORM_AXIS_REDUCE: return "vm_axis_reduce_kernel launch";
    default:
      snprintf(buf, sizeof(buf), "vm_elementwise_kernel%s launch (ndim=%d blocks=%lld smem=%zu n_regs=%d n_pf=%d n_insns=%d)", pl.lean ? " (lean)" : "", P.ndim,
               pl.blocks, pl.smem, P.n_regs, P.n_pf, P.n_insns);
  }
  return buf;
}

// Launches the plan's kernel and, for an axis reduction whose kernel writes fewer splits than requested, fills the rest
// with the identity.  No choices are made here.
static int launch(Plan& pl, cudaStream_t stream) {
  const KParams& P = pl.k;
  const unsigned blocks = (unsigned)pl.blocks;
  cudaError_t e = cudaSuccess;
  switch (pl.form) {
    case FORM_NONE: return 0;
    case FORM_TILE: e = launch_stencil_tile(pl.tile, stream); break;
    case FORM_STREAM: e = launch_stream(pl.stream, stream); break;
    case FORM_RNG: e = launch_rng(pl.rng, stream); break;
    case FORM_AXIS_AS_1D: e = launch_vm_elementwise_ax1d(P, blocks, pl.smem, stream); break;
    case FORM_AXIS_REDUCE: e = launch_vm_axis_reduce(P, blocks, pl.smem, stream); break;
    case FORM_ELEMENTWISE:
      switch (P.ndim) {
        case 1: e = pl.lean ? launch_vm_elementwise_lean(P, blocks, pl.smem, stream) : launch_vm_elementwise_nd1(P, blocks, pl.smem, stream); break;
        case 2: e = launch_vm_elementwise_nd2(P, blocks, pl.smem, stream); break;
        case 3: e = launch_vm_elementwise_nd3(P, blocks, pl.smem, stream); break;
        default: e = launch_vm_elementwise_nd5(P, blocks, pl.smem, stream); break;
      }
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
  if (pl.form == FORM_NONE) return "kernel=none";
  const char* form = pl.form == FORM_ELEMENTWISE ? "elementwise" : pl.form == FORM_AXIS_AS_1D ? "axis_as_1d" : "axis_reduce";
  const char* tiling = pl.form != FORM_ELEMENTWISE || op->ndim == 1 ? "" : pl.k.row_chunks > 0 ? " tiling=row" : " tiling=flat";
  char buf[200];
  snprintf(buf, sizeof(buf), "kernel=general_interpreter form=%s ndim=%d insns=%d views=%d%s ctas=%lld smem=%zu%s", form, op->ndim, op->n_insns,
           op->n_views, tiling, pl.blocks, pl.smem, pl.lean ? " variant=lean" : "");
  return buf;
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

extern "C" {

const char* rb200_last_error(void) { return g_last_error.c_str(); }
int rb200_abi_version(void) { return RB200_ABI_VERSION; }
int64_t rb200_launch_count(void) { return (int64_t)g_launches.load(); }
void rb200_reset_launch_count(void) { g_launches.store(0); }
int rb200_device_sm_count(void) { return sm_count(); }
int64_t rb200_red_scratch_bytes(void) { return (int64_t)(256 + 8 * RB200_MAX_REDS * kRedScratchPartials); }

int rb200_run_deferred_ops(const rb200_fused_op* op, void* stream_v) {
  bool empty = false;
  if (const int rc = validate(op, &empty)) return rc;
  if (empty) return 0;  // empty range: nothing to do
  // the op list is valid; from here on a device is needed (there is no CPU path)
  const int sms = sm_count();
  if (sms <= 0) return fail("no usable CUDA device (libramba_b200 has no CPU path)");
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
  const int sms = sm_count();
  if (sms <= 0) return fail("no usable CUDA device (libramba_b200 has no CPU path)");
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
  const int sms = sm_count();
  if (sms <= 0) return fail("no usable CUDA device (libramba_b200 has no CPU path)");
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
  const int sms = sm_count();
  if (sms <= 0) return fail("no usable CUDA device (libramba_b200 has no CPU path)");
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
  const int sms = sm_count();
  if (sms <= 0) return fail("no usable CUDA device (libramba_b200 has no CPU path)");
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
  const int sms = sm_count();
  if (sms <= 0) return fail("no usable CUDA device (libramba_b200 has no CPU path)");
  const cudaError_t e = launch_group(P, src_dtype, op, (const long long*)groups->offsets, (const long long*)groups->members, (const double*)center, out,
                                     scratch, (cudaStream_t)stream_v);
  if (e != cudaSuccess) return fail_cuda("group kernel launch", e);
  g_launches.fetch_add(1);
  return 0;
}

int rb200_reduce_partials(void* out, const void* partials, int64_t n, int64_t k, int64_t stride_k, int32_t dtype,
                          int32_t redop, void* stream_v) {
  if (!out || !partials) return fail("null pointer");
  if (n <= 0 || k <= 0) return 0;
  const int sms = sm_count();
  if (sms <= 0) return fail("no usable CUDA device (libramba_b200 has no CPU path)");
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
