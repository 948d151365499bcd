// rb200_plan.h — host-side planning rules that every kernel family shares (which operands are values, which views an op
// list reads and writes, the row-broadcast hoist, the row split of axis reductions, the global-reduction scratch), and
// the translation of op lists into the lean machine's LInsn records (rb200_lean.cuh).  The translation is 1:1 - same
// operation order, same compute classes - so a lean kernel and the general interpreter produce identical bits.
#pragma once
#include <string.h>

#include "rb200_lean.cuh"

namespace rb200 {

// Slot q (0: a, 1: b, 2: c) of I holds a value operand, except RED's b (the reduction slot) and SINCOS's c (the view the
// parked half is stored to).
static inline bool value_slot(const rb200_insn& I, int q) { return !(I.op == RB200_OP_RED && q == 1) && !(I.op == RB200_OP_SINCOS && q == 2); }

// the compute class an instruction fetches its value operands in: CVT fetches in the SOURCE class (imm & 0xff)
static inline int fetch_class(const rb200_insn& I) { return I.op == RB200_OP_CVT ? (int)(I.imm & 0xff) : (int)I.ctype; }

// Which views the op list reads as value operands, writes (stores and SINCOS's parked half) and stores under a mask.
struct ViewUse {
  bool read[RB200_MAX_VIEWS], written[RB200_MAX_VIEWS], masked[RB200_MAX_VIEWS];
};
static inline ViewUse view_use(const rb200_fused_op* op) {
  ViewUse u;
  memset(&u, 0, sizeof(u));
  for (int i = 0; i < op->n_insns; ++i) {
    const rb200_insn& I = op->insns[i];
    const uint8_t kinds[3] = {I.a_kind, I.b_kind, I.c_kind};
    const uint8_t idxs[3] = {I.a_idx, I.b_idx, I.c_idx};
    for (int q = 0; q < 3; ++q)
      if (kinds[q] == RB200_K_VIEW && value_slot(I, q)) u.read[idxs[q]] = true;
    if (I.op == RB200_OP_SINCOS && I.c_kind == RB200_K_VIEW) u.written[I.c_idx] = true;
    if (I.st_view != RB200_NOSTORE) {
      u.written[I.st_view] = true;
      if (I.mask_reg != RB200_NOSTORE) u.masked[I.st_view] = true;
    }
  }
  return u;
}

// Row-broadcast hoist over a [R][C] box: a view broadcast over the rows (strides {0, 1}) whose every value use fetches
// it in one compute class moves into a spill register, read once per column element instead of once per row.  Views
// are taken in order while fewer than max_hoist are hoisted and the next register (first_reg, first_reg + 1, ...) is
// below max_reg.  Rewrites the uses in insns; returns the number hoisted and, for each, its view, register and class.
static inline int hoist_row_broadcast(const rb200_fused_op* op, rb200_insn* insns, int first_reg, int max_reg, int max_hoist, int* view, int* reg,
                                      int* cls) {
  int n = 0;
  for (int v = 0; v < op->n_views && n < max_hoist && first_reg + n < max_reg; ++v) {
    if (op->views[v].stride[0] != 0 || op->views[v].stride[1] != 1) continue;
    int c = -1;
    bool same = true;
    for (int i = 0; i < op->n_insns; ++i) {
      const rb200_insn& I = insns[i];
      const uint8_t kinds[3] = {I.a_kind, I.b_kind, I.c_kind};
      const uint8_t idxs[3] = {I.a_idx, I.b_idx, I.c_idx};
      for (int q = 0; q < 3; ++q) {
        if (kinds[q] != RB200_K_VIEW || idxs[q] != v || !value_slot(I, q)) continue;
        if (I.op == RB200_OP_POWI && q == 1) same = false;  // an integer exponent operand
        if (c < 0) c = fetch_class(I);
        else if (c != fetch_class(I)) same = false;
      }
    }
    if (c < 0 || !same) continue;
    const int r = first_reg + n;
    view[n] = v;
    reg[n] = r;
    cls[n] = c;
    ++n;
    for (int i = 0; i < op->n_insns; ++i) {
      rb200_insn& I = insns[i];
      if (I.a_kind == RB200_K_VIEW && I.a_idx == v) { I.a_kind = RB200_K_REG; I.a_idx = (uint8_t)r; }
      if (I.b_kind == RB200_K_VIEW && I.b_idx == v && value_slot(I, 1)) { I.b_kind = RB200_K_REG; I.b_idx = (uint8_t)r; }
      if (I.c_kind == RB200_K_VIEW && I.c_idx == v && value_slot(I, 2)) { I.c_kind = RB200_K_REG; I.c_idx = (uint8_t)r; }
    }
  }
  return n;
}

// Row slices of an axis reduction whose columns take n_chunks CTAs: as many as `cap` CTAs allow, at most `want` and the
// row count, at least one.
static inline int row_split(long long cap, int n_chunks, int want, long long rows) {
  int s = (int)(cap / n_chunks);
  if (s > want) s = want;
  if ((long long)s > rows) s = (int)rows;
  return s < 1 ? 1 : s;
}

// An axis reduction's box: the first n_axis_red_dims dims are reduced (red_len rows), the others kept (kept elements);
// n_split: the row slices asked for, clamped to [1, red_len].
struct AxisBox {
  long long red_len, kept;
  int n_split;
};
static inline AxisBox axis_box(const rb200_fused_op* op) {
  AxisBox b = {1, 1, op->axis_nsplit};
  for (int d = 0; d < op->ndim; ++d) (d < op->n_axis_red_dims ? b.red_len : b.kept) *= op->itershape[d];
  if (b.n_split < 1) b.n_split = 1;
  if ((long long)b.n_split > b.red_len) b.n_split = (int)b.red_len;
  return b;
}

// Global reductions: red_scratch holds a ticket counter in its first kRedScratchHeader bytes, then the partials as
// [slot][CTA] for at most kRedScratchPartials CTAs (the grid cap of every launch with global reductions).
constexpr int kRedScratchPartials = 4096;
constexpr int kRedScratchHeader = 256;
constexpr long long kRedScratchBytes = kRedScratchHeader + 8ll * RB200_MAX_REDS * kRedScratchPartials;

// the op list's reduction slots
static inline void bind_reds(const rb200_fused_op* op, KRed* reds) {
  for (int s = 0; s < op->n_reds; ++s) {
    reds[s].op = op->reds[s].op;
    reds[s].ctype = op->reds[s].ctype;
    reds[s].out = op->reds[s].out;
    reds[s].out_dtype = op->reds[s].out_dtype;
  }
}
static inline void bind_red_scratch(const rb200_fused_op* op, unsigned int** counter, u64** partials) {
  *counter = (unsigned int*)op->red_scratch;
  *partials = (u64*)((char*)op->red_scratch + kRedScratchHeader);
}

// lean opcode of an op-list instruction (-1: not in the lean vocabulary)
static inline int lean_opcode(const rb200_fused_op* op, const rb200_insn& I) {
  switch (I.op) {
    case RB200_OP_MOV: return LO_MOV;
    case RB200_OP_ADD: return LO_ADD;
    case RB200_OP_SUB: return LO_SUB;
    case RB200_OP_MUL: return LO_MUL;
    case RB200_OP_DIV: return LO_DIV;
    case RB200_OP_NEG: return LO_NEG;
    case RB200_OP_ABS: return LO_ABS;
    case RB200_OP_SQUARE: return LO_SQUARE;
    case RB200_OP_MIN: return LO_MIN;
    case RB200_OP_MAX: return LO_MAX;
    case RB200_OP_MULADD: return LO_MULADD;
    case RB200_OP_MULSUB: return LO_MULSUB;
    case RB200_OP_MULRSUB: return LO_MULRSUB;
    case RB200_OP_RED: return LO_RED;
    case RB200_OP_POWI:  // x ** 2 with a scalar exponent is exactly x * x (Numba int_power)
      if (I.b_kind == RB200_K_SCAL && (long long)op->scalars[I.b_idx] == 2) return LO_SQUARE;
      return -1;
    case RB200_OP_CVT: {
      const int src = (int)(I.imm & 0xff);
      if ((I.imm >> 8) != 0) return -1;
      if (!(src == RB200_T_F64 || src == RB200_T_F32) || src == (int)I.ctype) return -1;
      return LO_CVT;
    }
    default: return -1;
  }
}

// float-arithmetic-only op list over float32/float64 views, no masks, no index operands
static inline bool lean_vocabulary_only(const rb200_fused_op* op, bool allow_red) {
  if (op->n_insns < 1) return false;
  for (int i = 0; i < op->n_views; ++i)
    if (op->views[i].dtype != RB200_F32 && op->views[i].dtype != RB200_F64) return false;
  for (int i = 0; i < op->n_insns; ++i) {
    const rb200_insn& I = op->insns[i];
    if (I.ctype != RB200_T_F64 && I.ctype != RB200_T_F32) return false;
    if (I.mask_reg != RB200_NOSTORE) return false;
    const int lop = lean_opcode(op, I);
    if (lop < 0) return false;
    if (lop == LO_RED && (!allow_red || I.ctype != RB200_T_F64)) return false;
    const uint8_t kinds[3] = {I.a_kind, I.b_kind, I.c_kind};
    for (int q = 0; q < 3; ++q)
      if (kinds[q] == RB200_K_IOTA && value_slot(I, q)) return false;
    if (I.a_kind == RB200_K_NONE) return false;
  }
  return true;
}

// insns (op's instructions, or a rewritten copy of them) into LInsn records.  view_kind[v] / view_arg[v]: how operand
// reads of view v are served (L_STAGED + staged-operand index, or L_DIRECT + direct-view index); stores always use
// store_arg[v] (index into the direct-view table)
static inline void lean_translate(const rb200_fused_op* op, const rb200_insn* insns, const int* view_kind, const int* view_arg, const int* store_arg,
                                  LInsn* out) {
  for (int i = 0; i < op->n_insns; ++i) {
    const rb200_insn& I = insns[i];
    LInsn L;
    memset(&L, 0, sizeof(L));
    int lop = lean_opcode(op, I);
    uint8_t kinds[3] = {I.a_kind, I.b_kind, I.c_kind};
    uint8_t idxs[3] = {I.a_idx, I.b_idx, I.c_idx};
    if (lop == LO_SQUARE || !value_slot(I, 1)) kinds[1] = RB200_K_NONE;  // (POWI's exponent is in the opcode)
    if ((lop == LO_ADD || lop == LO_MUL) && kinds[0] != RB200_K_ACC && kinds[1] == RB200_K_ACC) {
      kinds[1] = kinds[0]; idxs[1] = idxs[0];
      kinds[0] = RB200_K_ACC; idxs[0] = 0;
    } else if (lop == LO_SUB && kinds[0] != RB200_K_ACC && kinds[1] == RB200_K_ACC) {
      lop = LO_RSUB;  // b - a with a = the accumulator
      kinds[1] = kinds[0]; idxs[1] = idxs[0];
      kinds[0] = RB200_K_ACC; idxs[0] = 0;
    }
    unsigned char lk[3], la[3];
    for (int q = 0; q < 3; ++q) {
      switch (kinds[q]) {
        case RB200_K_ACC: lk[q] = L_ACC; la[q] = 0; break;
        case RB200_K_REG: lk[q] = L_REG; la[q] = idxs[q]; break;
        case RB200_K_SCAL: lk[q] = L_SCAL; la[q] = idxs[q]; break;
        case RB200_K_VIEW: lk[q] = (unsigned char)view_kind[idxs[q]]; la[q] = (unsigned char)view_arg[idxs[q]]; break;
        default: lk[q] = L_NONE; la[q] = 0;
      }
    }
    L.a_kind = lk[0]; L.a_arg = la[0];
    L.b_kind = lk[1]; L.b_arg = la[1];
    L.c_kind = lk[2]; L.c_arg = la[2];
    if (lop == LO_RED) {
      L.b_arg = I.b_idx;  // reduction slot
      L.red_op = (unsigned char)I.imm;
    }
    L.st_reg = I.st_reg;
    L.st_view = I.st_view == RB200_NOSTORE ? (unsigned char)RB200_NOSTORE : (unsigned char)store_arg[I.st_view];
    L.handler = (unsigned char)(lop * 4 + (I.ctype == RB200_T_F32 ? 2 : 0) + (L.a_kind == L_ACC ? 1 : 0));
    out[i] = L;
  }
}

// Fuse runs of add / sub / mul instructions whose right operand is a STAGED view and whose left operand is the running
// value into LO_CHAIN instructions (rb200_lean.cuh).  `insns` is rewritten in place; returns the new instruction count
// and fills `chain` (at most max_chain steps).
static inline int lean_fuse_chains(LInsn* insns, int n, LChainStep* chain, int max_chain, int* n_chain_out) {
  int out = 0, nc = 0;
  int i = 0;
  auto chain_op = [](const LInsn& L) -> int {
    const int lop = L.handler >> 2;
    return lop == LO_ADD ? LC_ADD : lop == LO_SUB ? LC_SUB : lop == LO_RSUB ? LC_RSUB : lop == LO_MUL ? LC_MUL : -1;
  };
  while (i < n) {
    const LInsn first = insns[i];
    int j = i;
    if (chain_op(first) >= 0 && first.b_kind == L_STAGED) {
      const int cls = (first.handler >> 1) & 1;
      j = i + 1;
      while (j < n && insns[j - 1].st_reg == RB200_NOSTORE && insns[j - 1].st_view == RB200_NOSTORE && chain_op(insns[j]) >= 0 &&
             insns[j].b_kind == L_STAGED && insns[j].a_kind == L_ACC && ((insns[j].handler >> 1) & 1) == cls && nc + (j - i) + 1 <= max_chain && (j - i) < 200)
        ++j;
      if (j - i >= 2) {
        LInsn L = first;
        L.handler = (unsigned char)(LO_CHAIN * 4 + cls * 2 + (first.a_kind == L_ACC ? 1 : 0));
        L.b_kind = L_NONE;
        L.b_arg = (unsigned char)nc;
        L.c_arg = (unsigned char)(j - i);
        L.st_reg = insns[j - 1].st_reg;
        L.st_view = insns[j - 1].st_view;
        for (int q = i; q < j; ++q) {
          chain[nc].op = (unsigned char)chain_op(insns[q]);
          chain[nc].staged = insns[q].b_arg;
          ++nc;
        }
        insns[out++] = L;
        i = j;
        continue;
      }
    }
    insns[out++] = first;
    ++i;
  }
  *n_chain_out = nc;
  return out;
}

}  // namespace rb200
