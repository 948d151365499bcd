// rb200_rng.cu — the random fill kernel: a plain draw (`rand(N)`, `normal(loc, scale, size)`, `randint(lo, hi, size)`)
// written straight to its array.  The general interpreter evaluates a PHILOX instruction once per element and keeps
// one lane of the block; here one thread computes a whole block (2 float64 / int64 or 4 float32 elements) and writes
// it with one 16-byte store, so a warp writes 512 consecutive bytes per step.  The values come from the same device
// functions (rb200_philox.h), so both paths give the same bits.  Write-only: itemsize bytes of HBM traffic per element.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "rb200_philox.h"
#include "rb200_rng.h"
#include "rb200_vm.cuh"

namespace rb200 {

namespace {

// one tail instruction `v (op) s`, rounded once like the interpreter's
__device__ __forceinline__ double rng_op(int o, double a, double b) {
  return o == RB200_OP_ADD ? __dadd_rn(a, b) : o == RB200_OP_SUB ? __dsub_rn(a, b) : __dmul_rn(a, b);
}
__device__ __forceinline__ float rng_op(int o, float a, float b) {
  return o == RB200_OP_ADD ? __fadd_rn(a, b) : o == RB200_OP_SUB ? __fsub_rn(a, b) : __fmul_rn(a, b);
}
__device__ __forceinline__ long long rng_op(int o, long long a, long long b) {
  return (long long)(o == RB200_OP_ADD ? (u64)a + (u64)b : o == RB200_OP_SUB ? (u64)a - (u64)b : (u64)a * (u64)b);
}

// the affine tail, instruction by instruction in the draw's class
template <class T> __device__ __forceinline__ T rng_tail(const RngParams& P, T v) {
#pragma unroll 1
  for (int q = 0; q < P.n_tail; ++q) v = rng_op(P.tail_op[q], v, CT<T>::get(P.tail_scal[q]));
  return v;
}

// FORM: rb200_philox_form; ND1: a 1-D range (one row, no index decoding)
template <int FORM, bool ND1> __global__ void __launch_bounds__(256) rng_fill_kernel(const __grid_constant__ RngParams P) {
  typedef typename std::conditional<FORM == RB200_PHILOX_UNIFORM32, float, typename std::conditional<FORM == RB200_PHILOX_INTEGER, long long, double>::type>::type T;
  constexpr int S = FORM == RB200_PHILOX_UNIFORM32 ? 2 : 1;  // log2 of the elements per block
  constexpr int E = 1 << S;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < P.items; t += stride) {
    long long row = 0, b = t;
    rng_u64 g0;  // linear index of the row's first element
    if constexpr (ND1) {
      g0 = (rng_u64)P.gstart[0];
    } else {
      row = t / P.per_row;
      b = t - row * P.per_row;
      long long rem = row, idx[RB200_MAX_DIMS];
#pragma unroll
      for (int d = RB200_MAX_DIMS - 2; d >= 0; --d) {
        if (d > P.ndim - 2) continue;
        const long long s = P.shape[d];
        const long long q = d == 0 ? 0 : rem / s;
        idx[d] = rem - q * s;
        rem = q;
      }
      g0 = (rng_u64)(P.gstart[0] + idx[0]);
#pragma unroll
      for (int d = 1; d < RB200_MAX_DIMS - 1; ++d)
        if (d <= P.ndim - 2) g0 = g0 * (rng_u64)P.mult[d] + (rng_u64)(P.gstart[d] + idx[d]);
      g0 = g0 * (rng_u64)P.mult[P.ndim - 1] + (rng_u64)P.gstart[P.ndim - 1];
    }
    const rng_u64 j = (g0 >> S) + (rng_u64)b;
    const long long lo = (long long)((j << S) - g0);  // row position of the block's first element (may be negative)
    if (lo >= P.inner) continue;                       // (per_row is an upper bound)
    const uint4 w = philox_block(j, P.key);
    rng_u64 v[E];
    if constexpr (FORM == RB200_PHILOX_UNIFORM32) {
      v[0] = CT<T>::bits(rng_tail<T>(P, philox_u01_32(w.x)));
      v[1] = CT<T>::bits(rng_tail<T>(P, philox_u01_32(w.y)));
      v[2] = CT<T>::bits(rng_tail<T>(P, philox_u01_32(w.z)));
      v[3] = CT<T>::bits(rng_tail<T>(P, philox_u01_32(w.w)));
    } else if constexpr (FORM == RB200_PHILOX_NORMAL64) {
      const double2 z = philox_normal_pair(w);
      v[0] = CT<T>::bits(rng_tail<T>(P, z.x));
      v[1] = CT<T>::bits(rng_tail<T>(P, z.y));
    } else if constexpr (FORM == RB200_PHILOX_INTEGER) {
      v[0] = CT<T>::bits(rng_tail<T>(P, philox_bounded(philox_half(w, 0), P.bound)));
      v[1] = CT<T>::bits(rng_tail<T>(P, philox_bounded(philox_half(w, 1), P.bound)));
    } else {
      v[0] = CT<T>::bits(rng_tail<T>(P, philox_u01_64(philox_half(w, 0))));
      v[1] = CT<T>::bits(rng_tail<T>(P, philox_u01_64(philox_half(w, 1))));
    }
    T* const rowp = reinterpret_cast<T*>(P.out) + row * P.inner;
    T* const p = rowp + lo;
    if (lo >= 0 && lo + E <= P.inner && (reinterpret_cast<uintptr_t>(p) & 15u) == 0) {
      if constexpr (E == 4) {
        *reinterpret_cast<uint4*>(p) = make_uint4((unsigned)v[0], (unsigned)v[1], (unsigned)v[2], (unsigned)v[3]);
      } else {
        *reinterpret_cast<ulonglong2*>(p) = make_ulonglong2(v[0], v[1]);
      }
    } else {
#pragma unroll
      for (int k = 0; k < E; ++k)
        if (lo + k >= 0 && lo + k < P.inner) p[k] = CT<T>::get(v[k]);
    }
  }
}

template <int FORM> cudaError_t launch_form(const RngPlan& T, cudaStream_t stream) {
  if (T.P.ndim == 1) rng_fill_kernel<FORM, true><<<(unsigned)T.blocks, 256, 0, stream>>>(T.P);
  else rng_fill_kernel<FORM, false><<<(unsigned)T.blocks, 256, 0, stream>>>(T.P);
  return cudaGetLastError();
}

const char* form_name(int f) {
  return f == RB200_PHILOX_UNIFORM64 ? "uniform64" : f == RB200_PHILOX_UNIFORM32 ? "uniform32" : f == RB200_PHILOX_NORMAL64 ? "normal64" : "integer";
}

}  // namespace

bool plan_rng(const rb200_fused_op* op, int sms, RngPlan& T) {
  const int nd = op->ndim;
  if (op->n_views != 1 || op->n_reds != 0 || op->n_axis_red_dims != 0 || op->n_insns < 1) return false;
  RngParams& P = T.P;
  memset(&P, 0, sizeof(P));
  P.ndim = nd;
  for (int d = 0; d < nd; ++d) {
    P.shape[d] = op->itershape[d];
    P.gstart[d] = op->global_start[d];
    P.mult[d] = 1;
  }
  // every instruction: no register, no mask; only the last one stores
  for (int i = 0; i < op->n_insns; ++i) {
    const rb200_insn& I = op->insns[i];
    if (I.st_reg != RB200_NOSTORE || I.mask_reg != RB200_NOSTORE) return false;
    if (I.st_view != (i == op->n_insns - 1 ? 0 : RB200_NOSTORE)) return false;
  }
  // the linear index in Horner form: MUL(IOTA 0, s1), ADD(ACC, IOTA 1), MUL(ACC, s2), ADD(ACC, IOTA 2), ...
  int pc = 0;
  if (nd > 1) {
    for (int d = 1; d < nd; ++d) {
      if (pc + 2 > op->n_insns) return false;
      const rb200_insn& M = op->insns[pc];
      const rb200_insn& A = op->insns[pc + 1];
      const bool m_ok = M.op == RB200_OP_MUL && M.ctype == RB200_T_I64 && M.b_kind == RB200_K_SCAL && M.c_kind == RB200_K_NONE &&
                        (d == 1 ? (M.a_kind == RB200_K_IOTA && M.a_idx == 0) : M.a_kind == RB200_K_ACC);
      const bool a_ok = A.op == RB200_OP_ADD && A.ctype == RB200_T_I64 && A.a_kind == RB200_K_ACC && A.b_kind == RB200_K_IOTA && A.b_idx == d &&
                        A.c_kind == RB200_K_NONE;
      if (!m_ok || !a_ok) return false;
      P.mult[d] = (long long)op->scalars[M.b_idx];
      pc += 2;
    }
  }
  if (pc >= op->n_insns) return false;
  const rb200_insn& X = op->insns[pc++];
  if (X.op != RB200_OP_PHILOX) return false;
  if (nd == 1 ? !(X.a_kind == RB200_K_IOTA && X.a_idx == 0) : X.a_kind != RB200_K_ACC) return false;
  P.form = (int)X.imm;
  P.key = op->scalars[X.b_idx];
  P.bound = P.form == RB200_PHILOX_INTEGER ? op->scalars[X.c_idx] : 1ull;
  const int cls = X.ctype;
  for (; pc < op->n_insns; ++pc) {
    const rb200_insn& I = op->insns[pc];
    if (P.n_tail >= kRngMaxTail) return false;
    if (!(I.op == RB200_OP_ADD || I.op == RB200_OP_SUB || I.op == RB200_OP_MUL) || I.ctype != cls || I.a_kind != RB200_K_ACC ||
        I.b_kind != RB200_K_SCAL || I.c_kind != RB200_K_NONE)
      return false;
    P.tail_op[P.n_tail] = I.op;
    P.tail_scal[P.n_tail] = op->scalars[I.b_idx];
    P.n_tail++;
  }
  // one view in the class's own dtype, contiguous (C order) over the range
  const rb200_view& v = op->views[0];
  const int own = cls == RB200_T_F64 ? RB200_F64 : cls == RB200_T_F32 ? RB200_F32 : RB200_I64;
  if (v.dtype != own) return false;
  long long expect = 1;
  for (int d = nd - 1; d >= 0; --d) {
    if (op->itershape[d] > 1 && v.stride[d] != expect) return false;
    expect *= op->itershape[d];
  }
  const int itemsize = cls == RB200_T_F32 ? 4 : 8;
  if (((uintptr_t)v.base) % itemsize != 0) return false;
  P.out = (char*)v.base;
  P.inner = op->itershape[nd - 1];
  P.rows = expect / (P.inner > 0 ? P.inner : 1);
  const int S = P.form == RB200_PHILOX_UNIFORM32 ? 2 : 1;
  const long long E = 1ll << S;
  if (nd == 1) {
    const unsigned long long g0 = (unsigned long long)P.gstart[0];
    P.per_row = (long long)(((g0 + (unsigned long long)P.inner - 1) >> S) - (g0 >> S) + 1);
  } else {
    P.per_row = (P.inner + 2 * (E - 1)) >> S;
  }
  P.items = P.rows * P.per_row;
  long long blocks = (P.items + 255) / 256;
  const long long cap = (long long)sms * 8;  // persistent grid: 8 CTAs of 256 threads fill an SM
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  T.blocks = blocks;
  return true;
}

std::string describe_rng(const RngPlan& T) {
  char buf[200];
  snprintf(buf, sizeof(buf), "kernel=rng_fill form=%s ndim=%d rows=%lld inner=%lld tail=%d ctas=%lld", form_name(T.P.form), T.P.ndim, T.P.rows,
           T.P.inner, T.P.n_tail, T.blocks);
  return buf;
}

cudaError_t launch_rng(const RngPlan& T, cudaStream_t stream) {
  switch (T.P.form) {
    case RB200_PHILOX_UNIFORM32: return launch_form<RB200_PHILOX_UNIFORM32>(T, stream);
    case RB200_PHILOX_NORMAL64: return launch_form<RB200_PHILOX_NORMAL64>(T, stream);
    case RB200_PHILOX_INTEGER: return launch_form<RB200_PHILOX_INTEGER>(T, stream);
    default: return launch_form<RB200_PHILOX_UNIFORM64>(T, stream);
  }
}

}  // namespace rb200
