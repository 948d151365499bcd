#pragma once
// rb200_interp.cuh — the op-list interpreter shared by the elementwise and axis-reduction kernels.
//
// Reference behaviour restated (not translated): the generated Numba loop body of
// ramba/ramba.py:8247-8265 executed by RemoteState.run_deferred_ops (ramba/ramba.py:3758-3780).
#include <cuda_runtime.h>
#include <math.h>
#include <type_traits>

#include "rb200_vm.cuh"
#include "rb200_handlers.h"
#include "rb200_philox.h"

namespace rb200 {

// one op-list instruction unpacked from its 16 bytes (two 8-byte constant-bank loads; fields that a
// path does not use cost nothing)
struct UInsn {
  uint2 lo, hi;
  __device__ __forceinline__ UInsn(const rb200_insn* p) {
    lo = *reinterpret_cast<const uint2*>(p);
    hi = *(reinterpret_cast<const uint2*>(p) + 1);
  }
  __device__ __forceinline__ unsigned op() const { return lo.x & 0xffu; }
  __device__ __forceinline__ unsigned ctype() const { return (lo.x >> 8) & 0xffu; }
  __device__ __forceinline__ unsigned a_kind() const { return (lo.x >> 16) & 0xffu; }
  __device__ __forceinline__ unsigned a_idx() const { return lo.x >> 24; }
  __device__ __forceinline__ unsigned b_kind() const { return lo.y & 0xffu; }
  __device__ __forceinline__ unsigned b_idx() const { return (lo.y >> 8) & 0xffu; }
  __device__ __forceinline__ unsigned c_kind() const { return (lo.y >> 16) & 0xffu; }
  __device__ __forceinline__ unsigned c_idx() const { return lo.y >> 24; }
  __device__ __forceinline__ unsigned st_reg() const { return hi.x & 0xffu; }
  __device__ __forceinline__ unsigned st_view() const { return (hi.x >> 8) & 0xffu; }
  __device__ __forceinline__ unsigned st2() const { return (hi.x >> 16) & 0xffu; }
  __device__ __forceinline__ unsigned mask_reg() const { return hi.x >> 24; }
  __device__ __forceinline__ unsigned imm() const { return hi.y; }
};

// compile-time unrolled loops over k with the shared-memory offset as an immediate
template <class T, int V, int K = 0> __device__ __forceinline__ void lds_vec64(unsigned base, T (&out)[V]) {
  if constexpr (K < V) {
    out[K] = CT<T>::get(lds64o<K * kThreads * 8>(base));
    lds_vec64<T, V, K + 1>(base, out);
  }
}
template <class T, int V, int K = 0> __device__ __forceinline__ void lds_vec32(unsigned base, T (&out)[V]) {  // float / int32 staged views
  if constexpr (K < V) {
    out[K] = CT<T>::get((u64)lds32o<K * kThreads * 4>(base));
    lds_vec32<T, V, K + 1>(base, out);
  }
}
template <int V, int K = 0> __device__ __forceinline__ void lds_vec32_as_f64(unsigned base, double (&out)[V]) {
  if constexpr (K < V) {
    out[K] = (double)__uint_as_float(lds32o<K * kThreads * 4>(base));
    lds_vec32_as_f64<V, K + 1>(base, out);
  }
}
template <int V, int K = 0> __device__ __forceinline__ void sts_vec64(unsigned base, const u64 (&v)[V]) {
  if constexpr (K < V) {
    sts64o<K * kThreads * 8>(base, v[K]);
    sts_vec64<V, K + 1>(base, v);
  }
}

// ---------------------------------------------------------------------------------------------
// Out-of-line store of the thread's V results for 1-D ops (one copy per compute class instead of one
// inlined copy per specialised handler: keeps the kernel small enough for the instruction cache and
// for ptxas).  Everything travels in registers: values as raw bits, the element offset of element 0
// and the per-k step.
template <class R>
__device__ __noinline__ void store_line(char* base, int dtype, long long off0, long long step, unsigned mask, u64 b0, u64 b1, u64 b2, u64 b3) {
  constexpr int V = 4;  // four elements per call; wider tiles call it once per group of four
  long long off[V] = {off0, off0 + step, off0 + 2 * step, off0 + 3 * step};
  R r[V] = {CT<R>::get(b0), CT<R>::get(b1), CT<R>::get(b2), CT<R>::get(b3)};
  constexpr int own = std::is_same<R, double>::value ? RB200_F64 : std::is_same<R, float>::value ? RB200_F32 : RB200_I64;
  if (dtype == own) {
    store_direct<R, R, V>(base, off, mask, r);
  } else if (dtype == RB200_BOOL) {
    long long b[V];
#pragma unroll
    for (int k = 0; k < V; ++k) b[k] = (r[k] != R(0)) ? 1 : 0;
    store_view<long long, V>(base, RB200_U8, off, mask, b);
  } else {
    store_view<R, V>(base, dtype, off, mask, r);
  }
}

// One converted store (any view dtype) of a value of compute class R
template <class R> __device__ __forceinline__ void store_one(char* base, int dtype, long long off, R x) {
  switch (dtype) {
    case RB200_F64: reinterpret_cast<double*>(base)[off] = (double)x; break;
    case RB200_F32: reinterpret_cast<float*>(base)[off] = (float)x; break;
    case RB200_I64: reinterpret_cast<long long*>(base)[off] = to_i64<R>(x); break;
    case RB200_I32: reinterpret_cast<int*>(base)[off] = to_storage<int>(x); break;
    default: store_narrow_one<R>(base, dtype, off, x);
  }
}

// Everything about a 1-D store that is not "full tile, contiguous, own dtype": write masks, ragged
// tiles, strided or converting views.  Out of line, one element at a time, the values handed over
// through the thread's scratch column in shared memory: the call sites in the specialised handlers
// stay small and need no extra registers (the hot loop is sensitive to both).
template <class R, int V>
__device__ __noinline__ void store_slow_1d(char* base, int dtype, long long stride, long long e0, unsigned valid, unsigned mask_addr,
                                           unsigned vals_addr) {
  const long long step = stride * kThreads;
  long long off = e0 * stride;
#pragma unroll 1
  for (int k = 0; k < V; ++k, off += step) {
    if (!((valid >> k) & 1u)) continue;
    if (mask_addr != 0xffffffffu && lds64(mask_addr + (unsigned)(k * kThreads * 8)) == 0ull) continue;
    store_one<R>(base, dtype, off, CT<R>::get(lds64(vals_addr + (unsigned)(k * kThreads * 8))));
  }
}

// N-d counterpart (V == 4): explicit element offsets
template <class R>
__device__ __noinline__ void store_slow_nd(char* base, int dtype, unsigned mask, long long o0, long long o1, long long o2, long long o3,
                                           unsigned vals_addr) {
  if (mask & 1u) store_one<R>(base, dtype, o0, CT<R>::get(lds64(vals_addr)));
  if (mask & 2u) store_one<R>(base, dtype, o1, CT<R>::get(lds64(vals_addr + (unsigned)(kThreads * 8))));
  if (mask & 4u) store_one<R>(base, dtype, o2, CT<R>::get(lds64(vals_addr + (unsigned)(2 * kThreads * 8))));
  if (mask & 8u) store_one<R>(base, dtype, o3, CT<R>::get(lds64(vals_addr + (unsigned)(3 * kThreads * 8))));
}

// ---------------------------------------------------------------------------------------------
// per-thread interpreter state.  ND = number of iteration dims this instantiation handles
// (ND == 1: collapsed 1-D op, the hot path; element k of the thread is e0 + k*256).
template <int V, int ND, bool LEAN = false> struct Ctx {
  static constexpr int kND = ND;
  const KParams& P;      // the __grid_constant__ kernel parameter: constant-bank (LDC) accesses
  unsigned regfile_s;    // shared-window byte address of this thread's column of the register file
  unsigned racc_s;       // this thread's accumulator of reduction slot 1 (slots 2.. follow at kThreads*8); global mode only
  unsigned pf_s;         // shared-window byte address of the current prefetch stage (element e of slot j at pf_s + j*V*2048 + e*itemsize)
  unsigned ocls_s;       // ND > 1: shared-window byte address of this thread's column of the offset-class table
  unsigned tid;
  long long e0;          // ND == 1: index of element 0 of this thread in the tile
  long long pe0;         // ND == 1, axis-as-1-D mode: e0 modulo the period of "periodic" (row-broadcast) views
  long long idx[V][ND];  // ND  > 1: N-d index of every element
  unsigned valid;        // bit k: element k exists
  u64 acc[V];

  __device__ __forceinline__ Ctx(const KParams& p) : P(p) {}

  // element offsets (in elements) of the thread's V elements inside view `vw`
  __device__ __forceinline__ void offsets(const KView& vw, long long (&off)[V]) const {
    if constexpr (ND == 1) {
      const long long s = vw.stride[0];
      const long long step = s * kThreads;  // uniform
      long long o = (vw.pf_slot == -2 ? pe0 : e0) * s;  // pf_slot -2: periodic view (broadcast over the reduced rows)
#pragma unroll
      for (int k = 0; k < V; ++k) {
        off[k] = o;
        o += step;
      }
    } else {
      const int c = vw.pf_slot;  // offset class: offsets were computed once for this tile
      if (c >= 0) {
        lds_vec64<long long, V>(ocls_s + (unsigned)(c * V * kThreads * 8), off);
        return;
      }
      compute_offsets(vw, off);
    }
  }
  __device__ __forceinline__ void compute_offsets(const KView& vw, long long (&off)[V]) const {
    if constexpr (ND > 1) {
#pragma unroll
      for (int k = 0; k < V; ++k) {
        long long o = 0;
#pragma unroll
        for (int d = 0; d < ND; ++d) o += idx[k][d] * vw.stride[d];
        off[k] = o;
      }
    }
  }
  // ND > 1: after the tile's indices are decoded, compute the element offsets of every offset class
  __device__ __forceinline__ void fill_offset_classes() {
    if constexpr (ND > 1) {
#pragma unroll 1
      for (int c = 0; c < P.n_ocls; ++c) {
        long long off[V];
        compute_offsets(P.views[P.ocls_view[c]], off);
        u64 b[V];
#pragma unroll
        for (int k = 0; k < V; ++k) b[k] = (u64)off[k];
        sts_vec64<V>(ocls_s + (unsigned)(c * V * kThreads * 8), b);
      }
    }
  }

  __device__ __forceinline__ unsigned reg_addr(int r, int k) const { return regfile_s + (unsigned)((r * V + k) * kThreads * 8); }
  __device__ __forceinline__ unsigned reg_base(int r) const { return regfile_s + (unsigned)(r * V * kThreads * 8); }

  template <class T> __device__ __forceinline__ void fetch(int kind, int i, T (&out)[V]) {
    switch (kind) {
      case RB200_K_ACC:
#pragma unroll
        for (int k = 0; k < V; ++k) out[k] = CT<T>::get(acc[k]);
        break;
      case RB200_K_REG:
#pragma unroll
        for (int k = 0; k < V; ++k) out[k] = CT<T>::get(lds64(reg_addr(i, k)));
        break;
      case RB200_K_VIEW: {
        const KView& vw = P.views[i];
        const int slot = vw.pf_slot;
        const int dt = vw.dtype;
        if (ND == 1 && slot >= 0) {  // (N-d kernels reuse pf_slot as the offset class)
          const unsigned slot_s = pf_s + (unsigned)(slot * V * kThreads * 8);
#pragma unroll
          for (int k = 0; k < V; ++k) out[k] = staged_load<T>(slot_s, k * kThreads + (int)tid, dt);
        } else {
          long long off[V];
          offsets(vw, off);
          load_view<T, V>(vw.base, dt, off, valid, out);
        }
      } break;
      case RB200_K_SCAL: {
        T s = CT<T>::get(P.scalars[i]);
#pragma unroll
        for (int k = 0; k < V; ++k) out[k] = s;
      } break;
      case RB200_K_IOTA: {
        if constexpr (ND == 1) {
          long long base = e0 + P.gstart[0];
#pragma unroll
          for (int k = 0; k < V; ++k) out[k] = (T)(base + (long long)k * kThreads);
        } else {
          long long g = 0;
#pragma unroll
          for (int d = 0; d < ND; ++d)
            if (d == i) g = P.gstart[d];
#pragma unroll
          for (int k = 0; k < V; ++k) {
            long long x = 0;
#pragma unroll
            for (int d = 0; d < ND; ++d)
              if (d == i) x = idx[k][d];
            out[k] = (T)(x + g);
          }
        }
      } break;
      default:
#pragma unroll
        for (int k = 0; k < V; ++k) out[k] = T(0);
    }
  }

  // store V results (already in registers as r[] and as raw bits in bits[]) into views[view]
  template <class R> __device__ __forceinline__ void store_out(int view, const R (&r)[V], const u64 (&bits)[V], unsigned m) {
    const KView& vw = P.views[view];
    if constexpr (ND == 1 && V % 4 == 0) {
      const long long st = vw.stride[0];
      const long long step = st * kThreads;
      char* const base = vw.base;
      const int dt = vw.dtype;
      constexpr int own1 = std::is_same<R, double>::value ? RB200_F64 : std::is_same<R, float>::value ? RB200_F32 : RB200_I64;
      if (dt == own1 && st == 1 && m == ((1u << V) - 1u)) {
        // full tile of a contiguous view in the result's own dtype: V coalesced stores at
        // immediate offsets from one address
        R* p = reinterpret_cast<R*>(base) + e0;
#pragma unroll
        for (int k = 0; k < V; ++k) stg<R>(p + k * kThreads, r[k]);
        return;
      }
#pragma unroll
      for (int g = 0; g < V / 4; ++g)
        store_line<R>(base, dt, (e0 + (long long)g * 4 * kThreads) * st, step, (m >> (4 * g)) & 0xfu, bits[4 * g], bits[4 * g + 1],
                      bits[4 * g + 2], bits[4 * g + 3]);
    } else {
      long long off[V];
      offsets(vw, off);
      constexpr int own = std::is_same<R, double>::value ? RB200_F64 : std::is_same<R, float>::value ? RB200_F32 : RB200_I64;
      if (vw.dtype == own) {
        store_direct<R, R, V>(vw.base, off, m, r);
      } else if (vw.dtype == RB200_BOOL) {
        long long b[V];
#pragma unroll
        for (int k = 0; k < V; ++k) b[k] = (r[k] != R(0)) ? 1 : 0;
        store_view<long long, V>(vw.base, RB200_U8, off, m, b);
      } else {
        store_view<R, V>(vw.base, vw.dtype, off, m, r);
      }
    }
  }

  // store V results (values r, raw bits b) to view `vi`, optionally masked by register `mreg`:
  // full contiguous tiles of the view's own dtype inline, everything else out of line
  template <class R> __device__ __forceinline__ void store_res(int vi, int mreg, const R (&r)[V], const u64 (&b)[V]) {
    if constexpr (LEAN) {
      // the lean kernel stores only unmasked, to contiguous views of the result's own dtype (host-checked)
      R* p = reinterpret_cast<R*>(P.views[vi].base) + e0;
      if (valid == ((1u << V) - 1u)) {
#pragma unroll
        for (int k = 0; k < V; ++k) stg<R>(p + k * kThreads, r[k]);
      } else {  // the ragged last tile
#pragma unroll
        for (int k = 0; k < V; ++k)
          if ((valid >> k) & 1u) stg<R>(p + k * kThreads, r[k]);
      }
    } else if constexpr (ND == 1 && (V == 4 || V == 8)) {
      const KView& vw = P.views[vi];
      constexpr int own1 = std::is_same<R, double>::value ? RB200_F64 : std::is_same<R, float>::value ? RB200_F32 : RB200_I64;
      const long long st = vw.stride[0];
      const bool plain = st == 1 && valid == ((1u << V) - 1u) && mreg == RB200_NOSTORE;
      if (plain && vw.dtype == own1) {
        R* p = reinterpret_cast<R*>(vw.base) + e0;
#pragma unroll
        for (int k = 0; k < V; ++k) stg<R>(p + k * kThreads, r[k]);
      } else if (std::is_same<R, double>::value && plain && vw.dtype == RB200_F32) {
        // float32 arrays computed in float64 (a Python float in the expression): the common converting store
        float* p = reinterpret_cast<float*>(vw.base) + e0;
#pragma unroll
        for (int k = 0; k < V; ++k) stg<float>(p + k * kThreads, (float)r[k]);
      } else {
        const unsigned maddr = mreg == RB200_NOSTORE ? 0xffffffffu : reg_base(mreg);
        sts_vec64<V>(reg_base(P.n_regs), b);  // scratch column behind the register file
        store_slow_1d<R, V>(vw.base, vw.dtype, st, e0, valid, maddr, reg_base(P.n_regs));
      }
    } else if constexpr (ND > 1 && V == 4) {
      const KView& vw = P.views[vi];
      constexpr int own = std::is_same<R, double>::value ? RB200_F64 : std::is_same<R, float>::value ? RB200_F32 : RB200_I64;
      long long off[V];
      offsets(vw, off);
      const bool plain = valid == 0xfu && mreg == RB200_NOSTORE;
      if (plain && vw.dtype == own) {
        R* p = reinterpret_cast<R*>(vw.base);
#pragma unroll
        for (int k = 0; k < V; ++k) stg<R>(p + off[k], r[k]);
      } else if (std::is_same<R, double>::value && plain && vw.dtype == RB200_F32) {
        float* p = reinterpret_cast<float*>(vw.base);
#pragma unroll
        for (int k = 0; k < V; ++k) stg<float>(p + off[k], (float)r[k]);
      } else {
        unsigned m = valid;
        if (mreg != RB200_NOSTORE) {
#pragma unroll
          for (int k = 0; k < V; ++k)
            if (lds64(reg_addr(mreg, k)) == 0ull) m &= ~(1u << k);
        }
        sts_vec64<V>(reg_base(P.n_regs), b);  // scratch column behind the register file
        store_slow_nd<R>(vw.base, vw.dtype, m, off[0], off[1], off[2], off[3], reg_base(P.n_regs));
      }
    } else {
      unsigned m = valid;
      if (mreg != RB200_NOSTORE) {
#pragma unroll
        for (int k = 0; k < V; ++k)
          if (lds64(reg_addr(mreg, k)) == 0ull) m &= ~(1u << k);
      }
      store_out<R>(vi, r, b, m);
    }
  }

  template <class R> __device__ __forceinline__ void finish(const UInsn& I, const R (&r)[V]) {
#pragma unroll
    for (int k = 0; k < V; ++k) acc[k] = CT<R>::bits(r[k]);
    if (I.st_reg() != RB200_NOSTORE) sts_vec64<V>(reg_base(I.st_reg()), acc);
    if (I.st_view() != RB200_NOSTORE) store_res<R>(I.st_view(), I.mask_reg(), r, acc);
  }
};

// rare ops: one out-of-line scalar routine each, called with static element indices so that the
// operand arrays never need dynamic indexing (which would push them to local memory)
template <class F> __device__ __noinline__ F rare_float_binary(int op, F a, F b) {
  return op == RB200_OP_FLOORDIV ? py_ffloordiv<F>(a, b) : op == RB200_OP_MOD ? py_fmod<F>(a, b) : (F)pow(a, b);
}
template <class F> __device__ __noinline__ F rare_powi(F a, long long e) { return powi<F>(a, e); }
template <class F> __device__ __noinline__ F rare_float_unary(int op, F x) {
  return op == RB200_OP_TAN    ? tan(x)
         : op == RB200_OP_SINH ? sinh(x)
         : op == RB200_OP_COSH ? cosh(x)
         : op == RB200_OP_TANH ? tanh(x)
         : op == RB200_OP_ASIN ? asin(x)
         : op == RB200_OP_ACOS ? acos(x)
         : op == RB200_OP_ATAN ? atan(x)
         : op == RB200_OP_EXP  ? exp(x)
         : op == RB200_OP_LOG  ? log(x)
                               : cbrt(x);
}
static __device__ __noinline__ long long rare_int_binary(int op, long long a, long long b) {
  return op == RB200_OP_FLOORDIV ? py_floordiv(a, b) : op == RB200_OP_MOD ? py_mod(a, b) : ipowi(a, b);
}

// ---------------------------------------------------------------------------------------------
// floating-point instruction set (F = double | float)
template <class F, int V, class C> __device__ __forceinline__ void exec_float(C& cx, const UInsn& I) {
  F a[V], b[V], r[V];
  long long p[V];
  const int op = I.op();
  cx.template fetch<F>(I.a_kind(), I.a_idx(), a);
  if (I.b_kind() != RB200_K_NONE && op != RB200_OP_POWI) cx.template fetch<F>(I.b_kind(), I.b_idx(), b);
  switch (op) {
    // ---- binary arithmetic.  __d*/__f*_rn: no FMA contraction across op-list instructions, every
    // op rounds once like the reference's separate scalar statements
    case RB200_OP_ADD:
#pragma unroll
      for (int k = 0; k < V; ++k) {
        if constexpr (sizeof(F) == 8) r[k] = __dadd_rn(a[k], b[k]);
        else r[k] = __fadd_rn(a[k], b[k]);
      }
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_SUB:
#pragma unroll
      for (int k = 0; k < V; ++k) {
        if constexpr (sizeof(F) == 8) r[k] = __dsub_rn(a[k], b[k]);
        else r[k] = __fsub_rn(a[k], b[k]);
      }
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_MUL:
#pragma unroll
      for (int k = 0; k < V; ++k) {
        if constexpr (sizeof(F) == 8) r[k] = __dmul_rn(a[k], b[k]);
        else r[k] = __fmul_rn(a[k], b[k]);
      }
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_DIV:
#pragma unroll
      for (int k = 0; k < V; ++k) {
        if constexpr (sizeof(F) == 8) r[k] = __ddiv_rn(a[k], b[k]);
        else r[k] = __fdiv_rn(a[k], b[k]);
      }
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_MIN:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = (b[k] < a[k]) ? b[k] : a[k];
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_MAX:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = (b[k] > a[k]) ? b[k] : a[k];
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_FLOORDIV:
    case RB200_OP_MOD:
    case RB200_OP_POW:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = rare_float_binary<F>(op, a[k], b[k]);
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_POWI: {
      long long e[V];
      cx.template fetch<long long>(I.b_kind(), I.b_idx(), e);
      bool sq = true;
#pragma unroll
      for (int k = 0; k < V; ++k) sq = sq && (e[k] == 2);
      if (sq) {  // x**2 == x*x exactly (int_power: r = 1*x*x)
#pragma unroll
        for (int k = 0; k < V; ++k) {
          if constexpr (sizeof(F) == 8) r[k] = __dmul_rn(a[k], a[k]);
          else r[k] = __fmul_rn(a[k], a[k]);
        }
      } else {
#pragma unroll
        for (int k = 0; k < V; ++k) r[k] = rare_powi<F>(a[k], e[k]);
      }
      cx.template finish<F>(I, r);
      return;
    }
    // ---- comparisons / logic -> bool (I64 class 0/1)
    case RB200_OP_GT:
    case RB200_OP_LT:
    case RB200_OP_GE:
    case RB200_OP_LE:
    case RB200_OP_EQ:
    case RB200_OP_NE:
#pragma unroll
      for (int k = 0; k < V; ++k) {
        F x = a[k], y = b[k];
        bool t = op == RB200_OP_GT ? x > y : op == RB200_OP_LT ? x < y : op == RB200_OP_GE ? x >= y : op == RB200_OP_LE ? x <= y : op == RB200_OP_EQ ? x == y : x != y;
        p[k] = t ? 1 : 0;
      }
      cx.template finish<long long>(I, p);
      return;
    case RB200_OP_LAND:
    case RB200_OP_LOR:
    case RB200_OP_LXOR:
#pragma unroll
      for (int k = 0; k < V; ++k) {
        bool x = a[k] != F(0), y = b[k] != F(0);
        p[k] = (op == RB200_OP_LAND ? (x && y) : op == RB200_OP_LOR ? (x || y) : (x != y)) ? 1 : 0;
      }
      cx.template finish<long long>(I, p);
      return;
    case RB200_OP_ISFINITE:
    case RB200_OP_ISINF:
    case RB200_OP_ISNAN:
    case RB200_OP_ISNEGINF:
    case RB200_OP_ISPOSINF:
    case RB200_OP_LNOT:
#pragma unroll
      for (int k = 0; k < V; ++k) {
        F x = a[k];
        bool t = op == RB200_OP_ISFINITE ? isfinite(x)
                 : op == RB200_OP_ISINF  ? isinf(x)
                 : op == RB200_OP_ISNAN  ? isnan(x)
                 : op == RB200_OP_ISNEGINF ? (isinf(x) && x < F(0))
                 : op == RB200_OP_ISPOSINF ? (isinf(x) && x > F(0))
                                           : (x == F(0));
        p[k] = t ? 1 : 0;
      }
      cx.template finish<long long>(I, p);
      return;
    // ---- unary
    case RB200_OP_MOV:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = a[k];
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_ABS:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = fabs(a[k]);
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_NEG:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = -a[k];
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_SQUARE:
#pragma unroll
      for (int k = 0; k < V; ++k) {
        if constexpr (sizeof(F) == 8) r[k] = __dmul_rn(a[k], a[k]);
        else r[k] = __fmul_rn(a[k], a[k]);
      }
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_SQRT:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = sqrt(a[k]);
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_SIN:
    case RB200_OP_COS:
    case RB200_OP_SINCOS: {
      F sn[V], cs[V];
      sincos_v<V>(a, sn, cs);
      const bool want_cos = (op == RB200_OP_COS) || (op == RB200_OP_SINCOS && I.imm());  // imm 1: accumulator half is cos
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = want_cos ? cs[k] : sn[k];
      if (op == RB200_OP_SINCOS) {
        u64 park[V];
        F parkv[V];
#pragma unroll
        for (int k = 0; k < V; ++k) {
          parkv[k] = want_cos ? sn[k] : cs[k];
          park[k] = CT<F>::bits(parkv[k]);
        }
        sts_vec64<V>(cx.reg_base(I.st2()), park);
        if (I.c_kind() == RB200_K_VIEW) cx.template store_out<F>(I.c_idx(), parkv, park, cx.valid);
      }
      cx.template finish<F>(I, r);
      return;
    }
    case RB200_OP_TAN:
    case RB200_OP_SINH:
    case RB200_OP_COSH:
    case RB200_OP_TANH:
    case RB200_OP_ASIN:
    case RB200_OP_ACOS:
    case RB200_OP_ATAN:
    case RB200_OP_EXP:
    case RB200_OP_LOG:
    case RB200_OP_CBRT:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = rare_float_unary<F>(op, a[k]);
      cx.template finish<F>(I, r);
      return;
    case RB200_OP_WHERE: {
      F c[V];
      cx.template fetch<F>(I.c_kind(), I.c_idx(), c);
      // condition arrives in `a`, already converted to the compute class (non-zero = true)
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = (a[k] != F(0)) ? b[k] : c[k];
      cx.template finish<F>(I, r);
      return;
    }
    case RB200_OP_MULADD:
    case RB200_OP_MULSUB:
    case RB200_OP_MULRSUB: {
      F c[V];
      cx.template fetch<F>(I.c_kind(), I.c_idx(), c);
      // product and sum round separately (two statements of the reference's loop body)
#pragma unroll
      for (int k = 0; k < V; ++k) {
        if constexpr (sizeof(F) == 8) {
          const double p = __dmul_rn(b[k], c[k]);
          r[k] = op == RB200_OP_MULADD ? __dadd_rn(a[k], p) : op == RB200_OP_MULSUB ? __dsub_rn(a[k], p) : __dsub_rn(p, a[k]);
        } else {
          const float p = __fmul_rn(b[k], c[k]);
          r[k] = op == RB200_OP_MULADD ? __fadd_rn(a[k], p) : op == RB200_OP_MULSUB ? __fsub_rn(a[k], p) : __fsub_rn(p, a[k]);
        }
      }
      cx.template finish<F>(I, r);
      return;
    }
    default: return;
  }
}

// integer instruction set (all integer arithmetic is int64, like Numba's intp promotion)
template <int V, class C> __device__ __forceinline__ void exec_int(C& cx, const UInsn& I) {
  long long a[V], b[V], r[V];
  cx.template fetch<long long>(I.a_kind(), I.a_idx(), a);
  if (I.b_kind() != RB200_K_NONE) cx.template fetch<long long>(I.b_kind(), I.b_idx(), b);
  const int op = I.op();
  switch (op) {
    case RB200_OP_MOV:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = a[k];
      break;
    case RB200_OP_ADD:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = a[k] + b[k];
      break;
    case RB200_OP_SUB:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = a[k] - b[k];
      break;
    case RB200_OP_MUL:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = a[k] * b[k];
      break;
    case RB200_OP_MIN:
    case RB200_OP_MAX:
    case RB200_OP_BAND:
    case RB200_OP_BOR:
    case RB200_OP_BXOR:
    case RB200_OP_SHL:
    case RB200_OP_SHR:
#pragma unroll
      for (int k = 0; k < V; ++k) {
        long long x = a[k], y = b[k];
        r[k] = op == RB200_OP_MIN ? ((y < x) ? y : x)
               : op == RB200_OP_MAX ? ((y > x) ? y : x)
               : op == RB200_OP_BAND ? (x & y)
               : op == RB200_OP_BOR  ? (x | y)
               : op == RB200_OP_BXOR ? (x ^ y)
               // counts outside [0, 63] shift every bit out, as NumPy's: 0, or -1 for a right shift of a negative x
               : op == RB200_OP_SHL  ? ((u64)y < 64 ? (long long)((u64)x << y) : 0)
                                     : ((u64)y < 64 ? (x >> y) : (x < 0 ? -1 : 0));
      }
      break;
    case RB200_OP_FLOORDIV:
    case RB200_OP_MOD:
    case RB200_OP_POWI:
    case RB200_OP_POW:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = rare_int_binary(op == RB200_OP_POW ? RB200_OP_POWI : op, a[k], b[k]);
      break;
    case RB200_OP_GT:
    case RB200_OP_LT:
    case RB200_OP_GE:
    case RB200_OP_LE:
    case RB200_OP_EQ:
    case RB200_OP_NE:
    case RB200_OP_LAND:
    case RB200_OP_LOR:
    case RB200_OP_LXOR:
#pragma unroll
      for (int k = 0; k < V; ++k) {
        long long x = a[k], y = b[k];
        bool t = op == RB200_OP_GT   ? x > y
                 : op == RB200_OP_LT ? x < y
                 : op == RB200_OP_GE ? x >= y
                 : op == RB200_OP_LE ? x <= y
                 : op == RB200_OP_EQ ? x == y
                 : op == RB200_OP_NE ? x != y
                 : op == RB200_OP_LAND ? (x != 0 && y != 0)
                 : op == RB200_OP_LOR  ? (x != 0 || y != 0)
                                       : ((x != 0) != (y != 0));
        r[k] = t ? 1 : 0;
      }
      break;
    case RB200_OP_ABS:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = a[k] < 0 ? -a[k] : a[k];
      break;
    case RB200_OP_NEG:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = -a[k];
      break;
    case RB200_OP_SQUARE:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = a[k] * a[k];
      break;
    case RB200_OP_INVERT:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = (I.imm() == 1) ? (a[k] == 0 ? 1 : 0) : ~a[k];  // imm 1: bool operand
      break;
    case RB200_OP_LNOT:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = a[k] == 0 ? 1 : 0;
      break;
    case RB200_OP_ISFINITE:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = 1;
      break;
    case RB200_OP_ISINF:
    case RB200_OP_ISNAN:
    case RB200_OP_ISNEGINF:
    case RB200_OP_ISPOSINF:
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = 0;
      break;
    case RB200_OP_WHERE: {
      long long c[V];
      cx.template fetch<long long>(I.c_kind(), I.c_idx(), c);
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = (a[k] != 0) ? b[k] : c[k];
    } break;
    case RB200_OP_MULADD:
    case RB200_OP_MULSUB:
    case RB200_OP_MULRSUB: {
      long long c[V];
      cx.template fetch<long long>(I.c_kind(), I.c_idx(), c);
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const long long p = b[k] * c[k];
        r[k] = op == RB200_OP_MULADD ? a[k] + p : op == RB200_OP_MULSUB ? a[k] - p : p - a[k];
      }
    } break;
    default: return;
  }
  cx.template finish<long long>(I, r);
}

// value a store + reload through integer storage dtype `dt` would give (wrap), as an int64
template <class T> __device__ __forceinline__ long long through_int(T x, int dt) {
  switch (dt) {
    case RB200_I32: return to_storage<int>(x);
    case RB200_BOOL: return x != T(0) ? 1 : 0;
    case RB200_U8: return to_storage<unsigned char>(x);
    case RB200_I8: return to_storage<signed char>(x);
    case RB200_I16: return to_storage<short>(x);
    case RB200_U16: return to_storage<unsigned short>(x);
    case RB200_U32: return to_storage<unsigned int>(x);
    default: return to_i64<T>(x);
  }
}

template <class S, int V, class C> __device__ __forceinline__ void exec_cvt_from(C& cx, const UInsn& I) {
  S a[V];
  cx.template fetch<S>(I.a_kind(), I.a_idx(), a);
  const int through = (int)(I.imm() >> 8);
  if (through - 1 == RB200_F64 || through - 1 == RB200_F32) {
#pragma unroll
    for (int k = 0; k < V; ++k) a[k] = through - 1 == RB200_F64 ? (S)(double)a[k] : (S)(float)a[k];
  } else if (through != 0) {
    // an integer storage dtype: the reloaded value is the wrapped integer itself, which the class of `a` (float32 above
    // 2^24) may not hold - go straight to the int64 class
    long long r[V];
#pragma unroll
    for (int k = 0; k < V; ++k) r[k] = through_int<S>(a[k], through - 1);
    cx.template finish<long long>(I, r);
    return;
  }
  switch (I.ctype()) {
    case RB200_T_F64: {
      double r[V];
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = (double)a[k];
      cx.template finish<double>(I, r);
    } break;
    case RB200_T_F32: {
      float r[V];
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = (float)a[k];
      cx.template finish<float>(I, r);
    } break;
    default: {
      long long r[V];
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = to_i64<S>(a[k]);
      cx.template finish<long long>(I, r);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// specialised handlers: operand kinds, compute class and opcode are template parameters; the host
// assigns one to every instruction whose operands are the accumulator, a spill register, a scalar
// or a staged (cp.async) view of the matching dtype (rb200_handlers.h).  For staged views the host
// has already replaced the view index by the prefetch slot.
template <class T, int SK, int V, class C> __device__ __forceinline__ void fetch_s(C& cx, int i, T (&out)[V]) {
  if constexpr (SK == S_ACC) {
#pragma unroll
    for (int k = 0; k < V; ++k) out[k] = CT<T>::get(cx.acc[k]);
  } else if constexpr (SK == S_REG) {
    lds_vec64<T, V>(cx.reg_base(i), out);
  } else if constexpr (SK == S_SCAL) {
    const T s = CT<T>::get(cx.P.scalars[i]);
#pragma unroll
    for (int k = 0; k < V; ++k) out[k] = s;
  } else if constexpr (SK == S_PFV) {  // staged view whose dtype is T's own storage type
    const unsigned slot_s = cx.pf_s + (unsigned)(i * V * kThreads * 8);
    if constexpr (sizeof(T) == 8) lds_vec64<T, V>(slot_s + cx.tid * 8u, out);
    else lds_vec32<T, V>(slot_s + cx.tid * 4u, out);
  } else if constexpr (SK == S_PFV32) {  // staged float32 view read in float64
    const unsigned slot_s = cx.pf_s + (unsigned)(i * V * kThreads * 8);
    if constexpr (std::is_same<T, double>::value) lds_vec32_as_f64<V>(slot_s + cx.tid * 4u, out);
  } else if constexpr (SK == S_VIEW) {  // direct view in T's own storage type
    const KView& vw = cx.P.views[i];
    long long off[V];
    cx.offsets(vw, off);
    load_direct<T, T, V>(vw.base, off, cx.valid, out);
  } else {  // S_VIEW32: direct float32 view read in float64
    const KView& vw = cx.P.views[i];
    long long off[V];
    cx.offsets(vw, off);
    if constexpr (std::is_same<T, double>::value) load_direct<double, float, V>(vw.base, off, cx.valid, out);
  }
}

template <int OP, class T, int AK, int BK, int V, class C> __device__ __forceinline__ void h_bin(C& cx, const UInsn& I) {
  T a[V], b[V], r[V];
  fetch_s<T, AK, V>(cx, I.a_idx(), a);
  fetch_s<T, BK, V>(cx, I.b_idx(), b);
#pragma unroll
  for (int k = 0; k < V; ++k) {
    if constexpr (sizeof(T) == 8 && !std::is_integral<T>::value) {
      r[k] = OP == RB200_OP_ADD ? __dadd_rn(a[k], b[k]) : OP == RB200_OP_SUB ? __dsub_rn(a[k], b[k]) : __dmul_rn(a[k], b[k]);
    } else if constexpr (sizeof(T) == 4) {
      r[k] = OP == RB200_OP_ADD ? __fadd_rn(a[k], b[k]) : OP == RB200_OP_SUB ? __fsub_rn(a[k], b[k]) : __fmul_rn(a[k], b[k]);
    } else {
      r[k] = OP == RB200_OP_ADD ? a[k] + b[k] : OP == RB200_OP_SUB ? a[k] - b[k] : a[k] * b[k];
    }
  }
  cx.template finish<T>(I, r);
}

template <int OP, class T, int AK, int V, class C> __device__ __forceinline__ void h_un(C& cx, const UInsn& I) {
  T a[V], r[V];
  fetch_s<T, AK, V>(cx, I.a_idx(), a);
  if constexpr (OP == RB200_OP_SIN || OP == RB200_OP_COS || OP == RB200_OP_SINCOS) {
    if constexpr (!std::is_integral<T>::value) {
      T sn[V], cs[V];
      sincos_v<V>(a, sn, cs);
      const bool want_cos = (OP == RB200_OP_COS) || (OP == RB200_OP_SINCOS && I.imm());
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = want_cos ? cs[k] : sn[k];
      if constexpr (OP == RB200_OP_SINCOS) {
        // the parked half goes to a spill register and, if c names a view, straight to that view
        u64 park[V];
        T parkv[V];
#pragma unroll
        for (int k = 0; k < V; ++k) {
          parkv[k] = want_cos ? sn[k] : cs[k];
          park[k] = CT<T>::bits(parkv[k]);
        }
        sts_vec64<V>(cx.reg_base(I.st2()), park);
        if (I.c_kind() == RB200_K_VIEW) cx.template store_res<T>(I.c_idx(), RB200_NOSTORE, parkv, park);
      }
    }
    cx.template finish<T>(I, r);
    return;
  }
#pragma unroll
  for (int k = 0; k < V; ++k) {
    if constexpr (OP == RB200_OP_MOV) r[k] = a[k];
    else if constexpr (OP == RB200_OP_NEG) r[k] = -a[k];
    else if constexpr (OP == RB200_OP_ABS) {
      if constexpr (std::is_integral<T>::value) r[k] = a[k] < 0 ? -a[k] : a[k];
      else r[k] = fabs(a[k]);
    } else if constexpr (OP == RB200_OP_SQUARE || OP == RB200_OP_POWI) {  // POWI here: exponent 2 (host-checked)
      if constexpr (std::is_integral<T>::value) r[k] = a[k] * a[k];
      else if constexpr (sizeof(T) == 8) r[k] = __dmul_rn(a[k], a[k]);
      else r[k] = __fmul_rn(a[k], a[k]);
    } else if constexpr (OP == RB200_OP_SQRT) r[k] = sqrt(a[k]);
    else if constexpr (OP == RB200_OP_SIN) r[k] = sin(a[k]);
    else if constexpr (OP == RB200_OP_COS) r[k] = cos(a[k]);
    else if constexpr (OP == RB200_OP_SINCOS) {
      T sn, cs;
      sincos(a[k], &sn, &cs);
      r[k] = I.imm() ? cs : sn;
      sts64(cx.reg_addr(I.st2(), k), CT<T>::bits(I.imm() ? sn : cs));
    }
  }
  cx.template finish<T>(I, r);
}

template <class TS, class TD, int AK, int V, class C> __device__ __forceinline__ void h_cvt(C& cx, const UInsn& I) {
  TS a[V];
  TD r[V];
  fetch_s<TS, AK, V>(cx, I.a_idx(), a);
#pragma unroll
  for (int k = 0; k < V; ++k) r[k] = to_storage<TD>(a[k]);  // float -> int64 by to_i64, not the saturating C cast
  cx.template finish<TD>(I, r);
}

template <class T, int AK, int V, bool AX, int NS, class C>
__device__ __forceinline__ void h_red(C& cx, const UInsn& I, u64 (&racc)[NS][AX ? V : 1]) {
  T a[V];
  fetch_s<T, AK, V>(cx, I.a_idx(), a);
  const int slot = I.b_idx();
  const int rop = (int)I.imm();
  if constexpr (!AX) {
    // fold the thread's V elements first (tree, no per-element branches), then one update of the
    // accumulator; elements past the end of the box are replaced by the identity
    const T ident = CT<T>::get(red_identity_bits(rop, std::is_integral<T>::value ? RB200_T_I64 : RB200_T_F64));
    if (cx.valid != ((1u << V) - 1u)) {
#pragma unroll
      for (int k = 0; k < V; ++k)
        if (!((cx.valid >> k) & 1u)) a[k] = ident;
    }
    // slot 0 lives in registers, the (rare) further slots of a multi-reduction op in shared memory
    if (rop == RB200_RED_ADD) {  // the common reduction: no per-combine operator test
#pragma unroll
      for (int w = V / 2; w >= 1; w >>= 1)
#pragma unroll
        for (int k = 0; k < w; ++k) a[k] = a[k] + a[k + w];
    } else {
#pragma unroll
      for (int w = V / 2; w >= 1; w >>= 1)
#pragma unroll
        for (int k = 0; k < w; ++k) a[k] = red_combine<T>(rop, a[k], a[k + w]);
    }
    if (slot == 0) {
      racc[0][0] = CT<T>::bits(red_combine<T>(rop, CT<T>::get(racc[0][0]), a[0]));
    } else {
      const unsigned addr = cx.racc_s + (unsigned)(slot - 1) * (unsigned)(kThreads * 8);
      sts64(addr, CT<T>::bits(red_combine<T>(rop, CT<T>::get(lds64(addr)), a[0])));
    }
  } else {
#pragma unroll
    for (int s = 0; s < NS; ++s)
      if (s == slot) {
#pragma unroll
        for (int k = 0; k < V; ++k)
          if ((cx.valid >> k) & 1u) {
            u64& t = racc[s][k];
            t = CT<T>::bits(red_combine<T>(rop, CT<T>::get(t), a[k]));
          }
      }
  }
}

// PHILOX: every element computes the block it reads (rb200_philox.h) and keeps its own lane of it
template <class R, int V, class C> __device__ __forceinline__ void finish_bits(C& cx, const UInsn& I, const u64 (&b)[V]) {
  R r[V];
#pragma unroll
  for (int k = 0; k < V; ++k) r[k] = CT<R>::get(b[k]);
  cx.template finish<R>(I, r);
}
template <int V, class C> __device__ __forceinline__ void exec_philox(C& cx, const UInsn& I) {
  long long a[V];
  cx.template fetch<long long>(I.a_kind(), I.a_idx(), a);
  const u64 key = cx.P.scalars[I.b_idx()];
  const u64 n = I.c_kind() == RB200_K_SCAL ? cx.P.scalars[I.c_idx()] : 1ull;
  const unsigned form = I.imm();
  u64 b[V];
#pragma unroll
  for (int k = 0; k < V; ++k) b[k] = philox_element_bits(a[k], key, n, form);
  switch (I.ctype()) {
    case RB200_T_F64: finish_bits<double, V>(cx, I, b); break;
    case RB200_T_F32: finish_bits<float, V>(cx, I, b); break;
    default: finish_bits<long long, V>(cx, I, b);
  }
}

// the generic path of one instruction (any opcode, class and operand kinds)
template <int V, bool AX, int NS, class C> __device__ __forceinline__ void generic_body(C& cx, const UInsn& I, u64 (&racc)[NS][AX ? V : 1]) {
  if (I.op() == RB200_OP_PHILOX) {
    exec_philox<V>(cx, I);
    return;
  }
  if (I.op() == RB200_OP_CVT) {
    switch (I.imm() & 0xff) {
      case RB200_T_F64: exec_cvt_from<double, V>(cx, I); break;
      case RB200_T_F32: exec_cvt_from<float, V>(cx, I); break;
      default: exec_cvt_from<long long, V>(cx, I);
    }
    return;
  }
  if (I.op() == RB200_OP_RED) {
    const int slot = I.b_idx();
    const int rop = (int)I.imm();
    if (I.ctype() == RB200_T_F64) {
      double a[V];
      cx.template fetch<double>(I.a_kind(), I.a_idx(), a);
      if constexpr (AX) {
#pragma unroll
        for (int s = 0; s < NS; ++s)
          if (s == slot) {
#pragma unroll
            for (int k = 0; k < V; ++k)
              if ((cx.valid >> k) & 1u) {
                u64& t = racc[s][AX ? k : 0];
                t = CT<double>::bits(red_combine<double>(rop, CT<double>::get(t), a[k]));
              }
          }
      } else {
        const unsigned addr = cx.racc_s + (unsigned)(slot - 1) * (unsigned)(kThreads * 8);
        u64 t = slot == 0 ? racc[0][0] : lds64(addr);
#pragma unroll
        for (int k = 0; k < V; ++k)
          if ((cx.valid >> k) & 1u) t = CT<double>::bits(red_combine<double>(rop, CT<double>::get(t), a[k]));
        if (slot == 0) racc[0][0] = t;
        else sts64(addr, t);
      }
    } else {
      long long a[V];
      cx.template fetch<long long>(I.a_kind(), I.a_idx(), a);
      if constexpr (AX) {
#pragma unroll
        for (int s = 0; s < NS; ++s)
          if (s == slot) {
#pragma unroll
            for (int k = 0; k < V; ++k)
              if ((cx.valid >> k) & 1u) {
                u64& t = racc[s][AX ? k : 0];
                t = (u64)red_combine<long long>(rop, (long long)t, a[k]);
              }
          }
      } else {
        const unsigned addr = cx.racc_s + (unsigned)(slot - 1) * (unsigned)(kThreads * 8);
        u64 t = slot == 0 ? racc[0][0] : lds64(addr);
#pragma unroll
        for (int k = 0; k < V; ++k)
          if ((cx.valid >> k) & 1u) t = (u64)red_combine<long long>(rop, (long long)t, a[k]);
        if (slot == 0) racc[0][0] = t;
        else sts64(addr, t);
      }
    }
    return;
  }
  switch (I.ctype()) {
    case RB200_T_F64: exec_float<double, V>(cx, I); break;
    case RB200_T_F32: exec_float<float, V>(cx, I); break;
    default: exec_int<V>(cx, I);
  }
}

#ifndef RB200_NO_FAST_HANDLERS
// Out of line in the kernels that have specialised handlers: the generic path needs several operand
// arrays at once, and inlined it would set the register allocation of the whole dispatch loop.  The
// interpreter state travels by value, the results come back through two small local arrays.
template <int V, bool AX, int NS, class C> __device__ __noinline__ void generic_step(C cx, int pc, u64* acc_out, u64* racc_io) {
  u64 racc[NS][AX ? V : 1];
#pragma unroll
  for (int s = 0; s < NS; ++s)
#pragma unroll
    for (int k = 0; k < (AX ? V : 1); ++k) racc[s][k] = racc_io[s * (AX ? V : 1) + k];
  const UInsn I(&cx.P.insns[pc]);
  generic_body<V, AX, NS>(cx, I, racc);
#pragma unroll
  for (int k = 0; k < V; ++k) acc_out[k] = cx.acc[k];
#pragma unroll
  for (int s = 0; s < NS; ++s)
#pragma unroll
    for (int k = 0; k < (AX ? V : 1); ++k) racc_io[s * (AX ? V : 1) + k] = racc[s][k];
}
#endif

// one interpreter pass over the op list for the thread's V elements.
// racc: reduction accumulators (raw bits), [slot][0] (global mode, AX=false) or [slot][k] (axis mode)
// NS = number of reduction slots carried in registers
template <int V, bool AX, int NS, bool LEAN = false, class C> __device__ __forceinline__ void run_program(C& cx, u64 (&racc)[NS][AX ? V : 1]) {
  const KParams& P = cx.P;
  const int n = P.n_insns;
  const unsigned valid_tile = cx.valid;
#pragma unroll 1
  for (int pc = 0; pc < n; ++pc) {
    const UInsn I(&P.insns[pc]);
    {
      // opaque per-instruction copy of the tile's element mask: keeps the compiler from hoisting the
      // per-bit tests of the rare paths out of this loop into eight more live registers
      unsigned v = valid_tile;
      // (1-D kernels only: the N-d kernels predicate every direct view load with these bits and are better off
      // with the hoisted tests)
      if constexpr (C::kND == 1) asm volatile("" : "+r"(v));
      cx.valid = v;
    }
#ifndef RB200_NO_FAST_HANDLERS
    const int h = P.handler[pc];
    if constexpr (LEAN) {  // lean handler ids (kLeanOf1); the host admits no instruction outside the lean set
#include "rb200_handlers_lean.inc"
    } else {
      if (h != H_GENERIC) {
#if RB200_HANDLER_SET == 2
#include "rb200_handlers_set2.inc"
#else
#include "rb200_handlers_set1.inc"
#endif
        continue;
      }
      {
        u64 acc_tmp[V], racc_tmp[NS * (AX ? V : 1)];
#pragma unroll
        for (int s = 0; s < NS; ++s)
#pragma unroll
          for (int k = 0; k < (AX ? V : 1); ++k) racc_tmp[s * (AX ? V : 1) + k] = racc[s][k];
        generic_step<V, AX, NS, C>(cx, pc, acc_tmp, racc_tmp);
#pragma unroll
        for (int k = 0; k < V; ++k) cx.acc[k] = acc_tmp[k];
#pragma unroll
        for (int s = 0; s < NS; ++s)
#pragma unroll
          for (int k = 0; k < (AX ? V : 1); ++k) racc[s][k] = racc_tmp[s * (AX ? V : 1) + k];
      }
    }
#else
    generic_body<V, AX, NS>(cx, I, racc);
#endif
  }
}

// decode a flat (row-major) element index into the N-d index, dims d0..ND-1 (d0 = first kept dim)
template <int ND> __device__ __forceinline__ void decode_index(const KParams& P, long long e, int d0, long long (&idx)[ND]) {
#pragma unroll
  for (int d = ND - 1; d >= 0; --d) {
    if (d >= P.ndim || d < d0) {
      if (d < d0) continue;
      idx[d] = 0;
      continue;
    }
    if (d == d0) {
      idx[d] = e;
    } else {
      const long long sd = P.shape[d];
      long long q;
      if (((e | sd) >> 31) == 0) q = (long long)((unsigned)e / (unsigned)sd);
      else q = e / sd;
      idx[d] = e - q * sd;
      e = q;
    }
  }
}

}  // namespace rb200
