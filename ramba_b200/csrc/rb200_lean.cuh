// rb200_lean.cuh — the "lean" op-list machine shared by the stencil/tile kernel (rb200_tile.cu) and the streaming
// kernel (rb200_stream.cu).
//
// The general interpreter (rb200_interp.cuh) pays ~40 instructions per dispatch for its generality (ten storage dtypes,
// three compute classes, masks, index operands, transcendental handlers).  Fused ops made of plain float arithmetic -
// the weighted shifted sums of stencils (ramba/ramba.py:8146-8188), affine maps feeding a reduction
// (ramba/ramba.py:5798-5814) - do not need any of that, and they are the ones that have to run at HBM speed with 4-byte
// elements.  The host translates such an op list 1:1 into LInsn records (same operation order, same compute classes,
// separate roundings: results are bit-identical to the general interpreter and the oracle); the kernels walk them with
// warp-uniform control flow only:
//   * the accumulator lives in registers (V elements per thread), spill registers in shared memory;
//   * one `switch` per instruction selects a handler instantiated for (operation, class, "a is the accumulator");
//     the remaining operands are fetched through a small uniform switch on their kind;
//   * a view operand is either STAGED (an element of a shared-memory tile: offset known per instruction) or DIRECT
//     (global memory, address affine in the element number).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "rb200_vm.cuh"

namespace rb200 {

constexpr int LV = 8;  // elements per thread per tile (256 threads -> 2048 elements)

enum LeanKind { L_ACC = 0, L_REG = 1, L_SCAL = 2, L_STAGED = 3, L_DIRECT = 4, L_NONE = 7 };
enum LeanOp {
  LO_MOV = 0, LO_ADD, LO_SUB, LO_RSUB, LO_MUL, LO_DIV, LO_NEG, LO_ABS, LO_SQUARE, LO_MIN, LO_MAX,
  LO_MULADD, LO_MULSUB, LO_MULRSUB, LO_CVT, LO_RED, LO_CHAIN, LO_NUM
};

struct LInsn {  // 12 bytes, read from the constant bank
  unsigned char handler;  // lean op * 4 + (f32 ? 2 : 0) + (a is the accumulator ? 1 : 0)
  unsigned char a_kind, b_kind, c_kind;
  unsigned char a_arg, b_arg, c_arg;
  unsigned char st_reg;   // RB200_NOSTORE: none
  unsigned char st_view;  // RB200_NOSTORE: none
  unsigned char red_op;   // LO_RED: rb200_redop; arg a_arg... slot in b_arg
  unsigned char pad[2];
};

// LO_CHAIN: `acc = (((a op1 s1) op2 s2) ...)` over STAGED operands - a run of add / sub / mul instructions of one class
// whose left operand is the running value (the neighbour sum of a stencil) executed by ONE dispatch: b_arg = first
// step in the kernel's chain table, c_arg = number of steps.  Same order, same roundings as the separate instructions.
enum LeanChainOp { LC_ADD = 0, LC_SUB = 1, LC_RSUB = 2, LC_MUL = 3 };
struct LChainStep {
  unsigned char op, staged, pad[2];
};

struct LDirect {  // a view addressed in global memory: element (z, y, x) at base + z*s0 + y*s1 + x*s2 (elements)
  char* base;
  long long s0, s1, s2;
  int dtype;  // RB200_F32 / RB200_F64
  int pad;
};

// N elements of a direct view, element k at element offset off + k * step; elements outside `valid` read as 0
template <class F, int N>
__device__ __forceinline__ void ldirect_load(const LDirect& v, long long off, long long step, unsigned valid, F (&out)[N]) {
  if (v.dtype == RB200_F32) {
    const float* p = reinterpret_cast<const float*>(v.base) + off;
#pragma unroll
    for (int k = 0; k < N; ++k, p += step) out[k] = ((valid >> k) & 1u) ? (F)ldg<float>(p) : F(0);
  } else {
    const double* p = reinterpret_cast<const double*>(v.base) + off;
#pragma unroll
    for (int k = 0; k < N; ++k, p += step) out[k] = ((valid >> k) & 1u) ? (F)ldg<double>(p) : F(0);
  }
}

// N values rounded to S, value k stored at p + k * step (step in units of *p: elements of S, or bytes for a char*);
// only elements inside `valid` are written.  full: all N are, one unpredicated loop.
template <class S, class F, int N, class Ptr>
__device__ __forceinline__ void store_strided(Ptr p, long long step, bool full, unsigned valid, const F (&r)[N]) {
  if (full) {
#pragma unroll
    for (int k = 0; k < N; ++k, p += step) stg<S>(reinterpret_cast<S*>(p), (S)r[k]);
  } else {
#pragma unroll
    for (int k = 0; k < N; ++k, p += step)
      if ((valid >> k) & 1u) stg<S>(reinterpret_cast<S*>(p), (S)r[k]);
  }
}

// the addressing of ldirect_load for a store, rounded to the view's dtype
template <class F, int N>
__device__ __forceinline__ void ldirect_store(const LDirect& v, long long off, long long step, unsigned valid, const F (&r)[N]) {
  if (v.dtype == RB200_F32) store_strided<float>(reinterpret_cast<float*>(v.base) + off, step, false, valid, r);
  else store_strided<double>(reinterpret_cast<double*>(v.base) + off, step, false, valid, r);
}

// the same store by byte address and byte step, with the unpredicated loop when all N elements are valid (the term
// kernels walk their output this way)
template <class F, int N> __device__ __forceinline__ void store_bytes(char* p, long long step, int dtype, unsigned valid, const F (&r)[N]) {
  constexpr unsigned all = N == 32 ? 0xffffffffu : (1u << N) - 1u;
  if (dtype == RB200_F32) store_strided<float>(p, step, valid == all, valid, r);
  else store_strided<double>(p, step, valid == all, valid, r);
}

// ---- register-level accumulator: low / high words kept apart so that float values cost one register
template <class F> struct LAcc;
template <> struct LAcc<double> {
  static __device__ __forceinline__ double get(unsigned lo, unsigned hi) { return __hiloint2double((int)hi, (int)lo); }
  static __device__ __forceinline__ void put(double v, unsigned& lo, unsigned& hi) {
    lo = (unsigned)__double2loint(v);
    hi = (unsigned)__double2hiint(v);
  }
};
template <> struct LAcc<float> {
  static __device__ __forceinline__ float get(unsigned lo, unsigned) { return __uint_as_float(lo); }
  static __device__ __forceinline__ void put(float v, unsigned& lo, unsigned&) { lo = __float_as_uint(v); }
};

template <class F> __device__ __forceinline__ F lean_lds(unsigned addr);
template <> __device__ __forceinline__ double lean_lds<double>(unsigned addr) { return __longlong_as_double((long long)lds64(addr)); }
template <> __device__ __forceinline__ float lean_lds<float>(unsigned addr) { return __uint_as_float(lds32(addr)); }
template <class F> __device__ __forceinline__ void lean_sts(unsigned addr, F v);
template <> __device__ __forceinline__ void lean_sts<double>(unsigned addr, double v) { sts64(addr, (u64)__double_as_longlong(v)); }
template <> __device__ __forceinline__ void lean_sts<float>(unsigned addr, float v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(__float_as_uint(v)) : "memory");
}

// a scalar operand (raw bits of its class) as a value of class F
template <class F> __device__ __forceinline__ F scal_as(u64 bits) {
  return sizeof(F) == 8 ? (F)__longlong_as_double((long long)bits) : (F)__uint_as_float((unsigned)bits);
}

// The operand kinds every lean kernel addresses alike: the accumulator (alo / ahi), a spill register (reg_s: this
// thread's column of the register file, 8-byte slots [reg][k][thread]) and a scalar.  A kernel's context derives from
// this and adds its staged and direct operands.
struct LeanRegs {
  unsigned reg_s;
  unsigned alo[LV], ahi[LV];

  template <class F> __device__ __forceinline__ void fetch_acc(F (&out)[LV]) const {
#pragma unroll
    for (int k = 0; k < LV; ++k) out[k] = LAcc<F>::get(alo[k], ahi[k]);
  }
  template <class F> __device__ __forceinline__ void fetch_reg(int reg, F (&out)[LV]) const {
    const unsigned addr = reg_s + (unsigned)reg * (LV * kThreads * 8);
#pragma unroll
    for (int k = 0; k < LV; ++k) out[k] = lean_lds<F>(addr + k * kThreads * 8);
  }
  template <class F> __device__ __forceinline__ void fetch_scal(u64 bits, F (&out)[LV]) const {
    const F s = scal_as<F>(bits);
#pragma unroll
    for (int k = 0; k < LV; ++k) out[k] = s;
  }
  template <class F> __device__ __forceinline__ void store_reg(int reg, const F (&r)[LV]) const {
    const unsigned addr = reg_s + (unsigned)reg * (LV * kThreads * 8);
#pragma unroll
    for (int k = 0; k < LV; ++k) lean_sts<F>(addr + k * kThreads * 8, r[k]);
  }
};

template <class F> struct LOther;
template <> struct LOther<double> { typedef float type; };
template <> struct LOther<float> { typedef double type; };

// one rounding per operation, never contracted
template <class F> __device__ __forceinline__ F l_add(F a, F b);
template <> __device__ __forceinline__ double l_add<double>(double a, double b) { return __dadd_rn(a, b); }
template <> __device__ __forceinline__ float l_add<float>(float a, float b) { return __fadd_rn(a, b); }
template <class F> __device__ __forceinline__ F l_sub(F a, F b);
template <> __device__ __forceinline__ double l_sub<double>(double a, double b) { return __dsub_rn(a, b); }
template <> __device__ __forceinline__ float l_sub<float>(float a, float b) { return __fsub_rn(a, b); }
template <class F> __device__ __forceinline__ F l_mul(F a, F b);
template <> __device__ __forceinline__ double l_mul<double>(double a, double b) { return __dmul_rn(a, b); }
template <> __device__ __forceinline__ float l_mul<float>(float a, float b) { return __fmul_rn(a, b); }
template <class F> __device__ __forceinline__ F l_div(F a, F b);
template <> __device__ __forceinline__ double l_div<double>(double a, double b) { return __ddiv_rn(a, b); }
template <> __device__ __forceinline__ float l_div<float>(float a, float b) { return __fdiv_rn(a, b); }

// ---------------------------------------------------------------------------------------------
// Handler body.  CX supplies: acc words alo/ahi[LV], fetch<F>(kind, arg, out), store_reg<F>(reg, r),
// store_view<F>(view, r), reduce<F>(slot, redop, r).
template <int LOP, class F, bool AACC, class CX> __device__ __forceinline__ void lean_exec(CX& cx, const LInsn& I) {
  F r[LV];
  if constexpr (LOP == LO_CVT) {
    typedef typename LOther<F>::type S;
    S s[LV];
    if constexpr (AACC) {
#pragma unroll
      for (int k = 0; k < LV; ++k) s[k] = LAcc<S>::get(cx.alo[k], cx.ahi[k]);
    } else {
      cx.template fetch<S>(I.a_kind, I.a_arg, s);
    }
#pragma unroll
    for (int k = 0; k < LV; ++k) r[k] = (F)s[k];
  } else {
    F a[LV];
    if constexpr (AACC) {
#pragma unroll
      for (int k = 0; k < LV; ++k) a[k] = LAcc<F>::get(cx.alo[k], cx.ahi[k]);
    } else {
      cx.template fetch<F>(I.a_kind, I.a_arg, a);
    }
    if constexpr (LOP == LO_MOV) {
#pragma unroll
      for (int k = 0; k < LV; ++k) r[k] = a[k];
    } else if constexpr (LOP == LO_CHAIN) {
#pragma unroll
      for (int k = 0; k < LV; ++k) r[k] = a[k];
#pragma unroll 1
      for (int s = 0; s < (int)I.c_arg; ++s) {
        F b[LV];
        const int cop = cx.template chain_fetch<F>((int)I.b_arg + s, b);
        if (cop == LC_ADD) {
#pragma unroll
          for (int k = 0; k < LV; ++k) r[k] = l_add<F>(r[k], b[k]);
        } else if (cop == LC_SUB) {
#pragma unroll
          for (int k = 0; k < LV; ++k) r[k] = l_sub<F>(r[k], b[k]);
        } else if (cop == LC_RSUB) {
#pragma unroll
          for (int k = 0; k < LV; ++k) r[k] = l_sub<F>(b[k], r[k]);
        } else {
#pragma unroll
          for (int k = 0; k < LV; ++k) r[k] = l_mul<F>(r[k], b[k]);
        }
      }
    } else if constexpr (LOP == LO_NEG) {
#pragma unroll
      for (int k = 0; k < LV; ++k) r[k] = -a[k];
    } else if constexpr (LOP == LO_ABS) {
#pragma unroll
      for (int k = 0; k < LV; ++k) r[k] = (F)fabs(a[k]);
    } else if constexpr (LOP == LO_SQUARE) {
#pragma unroll
      for (int k = 0; k < LV; ++k) r[k] = l_mul<F>(a[k], a[k]);
    } else if constexpr (LOP == LO_RED) {
      cx.template reduce<F>(I.b_arg, I.red_op, a);
      return;
    } else {
      F b[LV];
      cx.template fetch<F>(I.b_kind, I.b_arg, b);
      if constexpr (LOP == LO_ADD) {
#pragma unroll
        for (int k = 0; k < LV; ++k) r[k] = l_add<F>(a[k], b[k]);
      } else if constexpr (LOP == LO_SUB) {
#pragma unroll
        for (int k = 0; k < LV; ++k) r[k] = l_sub<F>(a[k], b[k]);
      } else if constexpr (LOP == LO_RSUB) {
#pragma unroll
        for (int k = 0; k < LV; ++k) r[k] = l_sub<F>(b[k], a[k]);
      } else if constexpr (LOP == LO_MUL) {
#pragma unroll
        for (int k = 0; k < LV; ++k) r[k] = l_mul<F>(a[k], b[k]);
      } else if constexpr (LOP == LO_DIV) {
#pragma unroll
        for (int k = 0; k < LV; ++k) r[k] = l_div<F>(a[k], b[k]);
      } else if constexpr (LOP == LO_MIN) {
#pragma unroll
        for (int k = 0; k < LV; ++k) r[k] = (b[k] < a[k]) ? b[k] : a[k];
      } else if constexpr (LOP == LO_MAX) {
#pragma unroll
        for (int k = 0; k < LV; ++k) r[k] = (b[k] > a[k]) ? b[k] : a[k];
      } else {
        F c[LV];
        cx.template fetch<F>(I.c_kind, I.c_arg, c);
#pragma unroll
        for (int k = 0; k < LV; ++k) {
          const F p = l_mul<F>(b[k], c[k]);
          r[k] = LOP == LO_MULADD ? l_add<F>(a[k], p) : LOP == LO_MULSUB ? l_sub<F>(a[k], p) : l_sub<F>(p, a[k]);
        }
      }
    }
  }
  if constexpr (LOP != LO_RED) {
#pragma unroll
    for (int k = 0; k < LV; ++k) LAcc<F>::put(r[k], cx.alo[k], cx.ahi[k]);
    if (I.st_reg != RB200_NOSTORE) cx.template store_reg<F>(I.st_reg, r);
    if (I.st_view != RB200_NOSTORE) cx.template store_view<F>(I.st_view, r);
  }
}

#define RB200_LEAN_CASE(LOP)                                             \
  case (LOP) * 4 + 0: lean_exec<LOP, double, false>(cx, I); break;       \
  case (LOP) * 4 + 1: lean_exec<LOP, double, true>(cx, I); break;        \
  case (LOP) * 4 + 2: lean_exec<LOP, float, false>(cx, I); break;        \
  case (LOP) * 4 + 3: lean_exec<LOP, float, true>(cx, I); break;

template <class CX> __device__ __forceinline__ void lean_dispatch(CX& cx, const LInsn& I) {
  switch (I.handler) {
    RB200_LEAN_CASE(LO_MOV)
    RB200_LEAN_CASE(LO_ADD)
    RB200_LEAN_CASE(LO_SUB)
    RB200_LEAN_CASE(LO_RSUB)
    RB200_LEAN_CASE(LO_MUL)
    RB200_LEAN_CASE(LO_DIV)
    RB200_LEAN_CASE(LO_NEG)
    RB200_LEAN_CASE(LO_ABS)
    RB200_LEAN_CASE(LO_SQUARE)
    RB200_LEAN_CASE(LO_MIN)
    RB200_LEAN_CASE(LO_MAX)
    RB200_LEAN_CASE(LO_MULADD)
    RB200_LEAN_CASE(LO_MULSUB)
    RB200_LEAN_CASE(LO_MULRSUB)
    RB200_LEAN_CASE(LO_CVT)
    RB200_LEAN_CASE(LO_RED)
    RB200_LEAN_CASE(LO_CHAIN)
    default: break;
  }
}

}  // namespace rb200
