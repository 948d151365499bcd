// rb200_interp_plan.cu — host-side plan of the general interpreter (rb200_elementwise*.cu, rb200_axis.cu): form, handler
// ids, staging, grid and shared memory of one op list.
#include <stdio.h>
#include <string.h>

#include <string>

#include "rb200_handlers.h"
#include "rb200_launch.h"
#include "rb200_plan.h"

namespace rb200 {

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

static void assign_handlers(KParams& P, const rb200_fused_op* op, int set) {
  for (int i = 0; i < P.n_insns; ++i) {
    rb200_insn I = P.insns[i];
    int h = H_GENERIC;
    int ai = I.a_idx, bi = I.b_idx;
    const int ak = static_kind(P, set, I.a_kind, &ai, fetch_class(I));
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
      if (value_slot(I, 1)) I.b_idx = (uint8_t)bi;
      P.insns[i] = I;
    }
    P.handler[i] = (unsigned short)h;
  }
}

// axis-as-1-D form: [R reduced rows][C kept elements], every view contiguous over the box or broadcast over the rows,
// C a multiple of the 1-D tile, one reduction slot, no index operands: the staged 1-D kernel with V column accumulators
// per thread (rb200_elementwise_ax1d.cu).  false: not of this form, or its shared memory does not fit.
static bool plan_axis_as_1d(const rb200_fused_op* op, int sms, const ViewUse& use, size_t reg_bytes, InterpPlan& pl) {
  const KParams& P = pl.k;
  const long long TILE1 = (long long)kThreads * kV1;
  const long long red_len = P.red_len, kept = P.total;
  bool ok = (op->ndim == 2 && P.red_ndim == 1 && op->n_reds == 1 && kept % TILE1 == 0 && kept / TILE1 <= (long long)sms * 2 && red_len >= 2);
  for (int i = 0; i < op->n_insns && ok; ++i) {
    const rb200_insn& I = op->insns[i];
    if (I.a_kind == RB200_K_IOTA || I.b_kind == RB200_K_IOTA || I.c_kind == RB200_K_IOTA) ok = false;
  }
  for (int i = 0; i < op->n_views && ok; ++i) {
    const rb200_view& v = op->views[i];
    if (use.written[i]) ok = false;  // stage 1 of an axis reduction only reads
    if (!use.read[i]) continue;
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
  const int n_split_eff = row_split((long long)sms * 2, n_chunks, P.n_split, red_len);
  Q.n_split_chunks = n_chunks;
  Q.n_split = n_split_eff;
  Q.red_len = kept;  // in this mode: elements per row (partials are [split][kept])
  Q.n_pf = 0;
  for (int i = 0; i < op->n_views; ++i) {
    KView& k = Q.views[i];
    const rb200_view& v = op->views[i];
    k.stride[0] = 1;
    k.pf_slot = -1;
    if (!use.read[i]) continue;
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
  Q.n_hoist = hoist_row_broadcast(op, Q.insns, Q.n_regs, RB200_MAX_REGS, kMaxPf, Q.hoist_view, Q.hoist_reg, Q.hoist_cls);
  Q.n_regs += Q.n_hoist;
  const size_t reg_bytes1 = (size_t)(Q.n_regs + 1) * V1 * kThreads * 8;
  Q.bulk = Q.n_pf > 0 ? 1 : 0;
  for (int j = 0; j < Q.n_pf; ++j)
    if ((((uintptr_t)op->views[Q.pf_view[j]].base) & 15u) != 0) Q.bulk = 0;
  Q.n_stages = 2;
  const size_t pf_bytes1 = (size_t)Q.n_pf * Q.n_stages * V1 * kThreads * 8;
  if (reg_bytes1 + pf_bytes1 > 200 * 1024) return false;  // does not fit: the general axis kernel runs it
  assign_handlers(Q, op, 1);
  pl.k = Q;
  pl.form = INTERP_AXIS_AS_1D;
  pl.blocks = (long long)n_split_eff * n_chunks;
  pl.smem = reg_bytes1 + pf_bytes1;
  pl.n_written = n_split_eff;
  return true;
}

// The lean 1-D kernel (rb200_elementwise_lean.cu) runs a 1-D op list, already staged and given its set-1 handlers, when
// every instruction has a handler of the lean set, nothing is reduced, every store is unmasked and goes to a contiguous
// view of the result's own dtype, and the staged views move by bulk copies: what the lean kernel leaves out (the generic
// path, reductions, converting / masked / strided stores, the per-thread staging pipeline) is then never needed.
static bool lean_interp_eligible(const KParams& P, const rb200_fused_op* op) {
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

void plan_interp(const rb200_fused_op* op, int sms, bool row_mode, bool lean, bool per_tile, InterpPlan& pl) {
  // the 1-D kernel owns 8 elements per thread, the N-d and axis kernels 4
  const int V = (op->ndim == 1 && op->n_axis_red_dims == 0) ? kV1 : kV;
  const long long TILE = (long long)kThreads * V;
  KParams& P = pl.k;
  memset(&P, 0, sizeof(P));
  pl.lean = false;
  pl.per_tile = false;
  pl.n_written = 0;
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
  const ViewUse use = view_use(op);
  for (int i = 0; i < op->n_insns; ++i) P.insns[i] = op->insns[i];
  for (int i = 0; i < op->n_scalars; ++i) P.scalars[i] = op->scalars[i];
  for (int i = 0; i < op->n_views; ++i) {
    const rb200_view& v = op->views[i];
    KView& k = P.views[i];
    k.base = (char*)v.base;
    k.dtype = v.dtype;
    k.pf_slot = -1;
    for (int d = 0; d < op->ndim; ++d) k.stride[d] = v.stride[d];
  }
  bind_reds(op, P.reds);
  const size_t reg_bytes = (size_t)(op->n_regs + 1) * V * kThreads * 8;  // + the scratch column of the out-of-line stores

  if (op->n_axis_red_dims != 0) {
    const AxisBox box = axis_box(op);
    P.red_ndim = op->n_axis_red_dims;
    P.red_len = box.red_len;
    P.n_split = box.n_split;
    P.red_split = (box.red_len + box.n_split - 1) / box.n_split;
    P.total = box.kept;
    P.n_tiles = ((box.kept + TILE - 1) / TILE) * box.n_split;
    P.red_partials = (u64*)op->red_scratch;
    if (plan_axis_as_1d(op, sms, use, reg_bytes, pl)) return;
    long long blocks = P.n_tiles;
    long long cap = (long long)sms * 4;
    if (blocks > cap) blocks = cap;
    pl.form = INTERP_AXIS_REDUCE;
    pl.blocks = blocks;
    pl.smem = reg_bytes;
    pl.n_written = box.n_split;
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
    if (row_mode && inner * 5 >= chunks * TILE * 4 && chunks < (1ll << 30)) {
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
      if (use.read[i] && !use.masked[i] && wide_ok && reg_bytes + (size_t)(P.n_pf + 1) * 2 * V * kThreads * 8 <= 108 * 1024) {
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
  if (lean && lean_interp_eligible(P, op)) {
    pl.lean = true;
    for (int i = 0; i < P.n_insns; ++i) P.handler[i] = kLeanOf1[P.handler[i]];
  }
  // (the lean kernel's stores never go through the scratch column behind the register file)
  const size_t smem = (pl.lean ? reg_bytes - (size_t)V * kThreads * 8 : reg_bytes) + pf_bytes + ocls_bytes;
  if (op->n_reds > 0) bind_red_scratch(op, &P.red_counter, &P.red_partials);
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
  // The lean kernel (no reductions) runs one CTA per tile: the kernel's walk then ends after one tile.  Write-heavy
  // streams reach HBM faster from CTAs issued in tile order than from a persistent grid walking tiles b, b+grid, ...
  // (the float64 sin/cos chain, 1 read / 3 writes: 11.45 -> 10.88 ms on an H100, DESIGN §8 item 4); each element keeps
  // its thread, so its bits do not change.
  pl.per_tile = pl.lean && per_tile;
  if (blocks > cap && !pl.per_tile) blocks = cap;
  pl.form = INTERP_ELEMENTWISE;
  pl.blocks = blocks;
  pl.smem = smem;
}

std::string describe_interp(const rb200_fused_op* op, const InterpPlan& pl) {
  const char* form = pl.form == INTERP_ELEMENTWISE ? "elementwise" : pl.form == INTERP_AXIS_AS_1D ? "axis_as_1d" : "axis_reduce";
  const char* tiling = pl.form != INTERP_ELEMENTWISE || op->ndim == 1 ? "" : pl.k.row_chunks > 0 ? " tiling=row" : " tiling=flat";
  char buf[220];
  snprintf(buf, sizeof(buf), "kernel=general_interpreter form=%s ndim=%d insns=%d views=%d%s ctas=%lld%s smem=%zu", form, op->ndim, op->n_insns,
           op->n_views, tiling, pl.blocks, pl.per_tile ? " grid=cta_per_tile" : "", pl.smem);
  std::string s = buf;
  // the instructions (by index) without a specialised handler, which take the generic decode path (the axis kernel runs
  // every instruction on it)
  if (pl.form != INTERP_AXIS_REDUCE)
    for (int i = 0, n = 0; i < pl.k.n_insns; ++i)
      if (pl.k.handler[i] == H_GENERIC) s += (n++ ? "," : " generic=") + std::to_string(i);
  if (pl.lean) s += " variant=lean";
  return s;
}

}  // namespace rb200
