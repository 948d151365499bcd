// rb200_vm.cuh — device side of the op-list accumulator machine (sm_90a): data layout, loads,
// stores and scalar op semantics.
//
// The reference's worker executes Python source generated per fused op and JIT-compiled by Numba
// (ramba/ramba.py:8247-8265, 3758-3780).  Here the same loop body is an op list that a hand-written
// CUDA kernel walks.  Work decomposition: a CTA of 256 threads owns one tile of 256*V consecutive
// elements of the (row-major, collapsed) iteration space at a time; thread t owns elements
// t, 256+t, 512+t, ... of the tile ("strided-V"), so every per-k access of a warp covers 32
// consecutive elements: fully coalesced requests for any contiguous view, with no alignment
// requirement on the view's base (slices starting at odd offsets run at the same speed).  The
// running value stays in registers (the accumulator); values needed later go to a shared-memory
// register file; read-only input views of 1-D (collapsed) ops are staged one tile ahead into shared
// memory with per-thread cp.async (LDGSTS) so that HBM latency overlaps the interpretation of the
// current tile.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "../../include/ramba_b200.h"

namespace rb200 {

typedef unsigned long long u64;

constexpr int kThreads = 256;
constexpr int kMaxD = RB200_MAX_DIMS;
constexpr int kMaxPf = 4;    // input views staged through shared memory
constexpr int kMaxOcls = 6;  // N-d kernels: distinct stride signatures whose element offsets are cached per tile

struct KView {
  char* base;
  long long stride[kMaxD];  // elements
  int dtype;
  int pf_slot;  // 1-D: >= 0: staged into prefetch slot pf_slot; -1: read directly; -2: read directly, periodic (axis-as-1-D)
                // N-d: >= 0: offset class (views with identical strides share per-tile element offsets); -1: none
};

struct KRed {
  int op, ctype;
  void* out;
  int out_dtype;
  int pad;
};

struct KParams {
  int ndim, n_insns, n_views, n_regs, n_reds, n_pf;
  int pf_view[kMaxPf];
  int wide;  // 1: element indices need 64 bits
  int bulk;  // 1: staged views are contiguous and 16-byte aligned -> whole tiles move by bulk async copy
  long long shape[kMaxD];
  long long gstart[kMaxD];
  long long total;    // elements of the (kept) iteration space
  long long n_tiles;  // ceil(total / (kThreads*V)); row mode: rows * row_chunks
  int row_chunks;     // N-d row mode (> 0): tiles per row of the innermost dim; a tile never crosses a row, the outer indices are per-tile
  // axis reduction (column form): leading red_ndim dims are walked sequentially
  long long red_len;
  long long red_split;
  int n_split;
  int red_ndim;
  int n_split_chunks;  // axis-as-1-D mode: column chunks (C / tile) = CTAs per split
  int n_stages;        // depth of the staging ring (2)
  // axis-as-1-D mode: row-broadcast ("periodic") views are loop invariant for a CTA — they are loaded
  // once into spill registers before the row loop
  int n_hoist;
  int n_ocls;  // N-d kernels: number of offset classes; ocls_view[c] = a view carrying class c's strides
  int ocls_view[kMaxOcls];
  int hoist_view[kMaxPf], hoist_reg[kMaxPf], hoist_cls[kMaxPf];
  KView views[RB200_MAX_VIEWS];
  u64 scalars[RB200_MAX_SCALARS];
  rb200_insn insns[RB200_MAX_INSNS];
  unsigned short handler[RB200_MAX_INSNS];  // specialised handler per instruction (rb200_handlers.h), 0 = generic
  KRed reds[RB200_MAX_REDS];
  u64* red_partials;
  unsigned int* red_counter;
};

// ---------------------------------------------------------------------------------------------
// raw 64-bit machine values <-> the three compute classes (register moves, never memory)
template <class T> struct CT;
template <> struct CT<double> {
  static __device__ __forceinline__ double get(u64 v) { return __longlong_as_double((long long)v); }
  static __device__ __forceinline__ u64 bits(double x) { return (u64)__double_as_longlong(x); }
};
template <> struct CT<float> {
  static __device__ __forceinline__ float get(u64 v) { return __uint_as_float((unsigned)v); }
  static __device__ __forceinline__ u64 bits(float x) { return (u64)__float_as_uint(x); }
};
template <> struct CT<long long> {
  static __device__ __forceinline__ long long get(u64 v) { return (long long)v; }
  static __device__ __forceinline__ u64 bits(long long x) { return (u64)x; }
};

// ---------------------------------------------------------------------------------------------
// shared memory by 32-bit shared-window address (guarantees LDS/STS, never generic LD/ST)
__device__ __forceinline__ u64 lds64(unsigned addr) {
  u64 v;
  asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
  return v;
}
// immediate-offset forms: one address register serves all V accesses of an operand
template <int OFF> __device__ __forceinline__ u64 lds64o(unsigned addr) {
  u64 v;
  asm volatile("ld.shared.u64 %0, [%1+%2];" : "=l"(v) : "r"(addr), "n"(OFF) : "memory");
  return v;
}
template <int OFF> __device__ __forceinline__ unsigned lds32o(unsigned addr) {
  unsigned v;
  asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(OFF) : "memory");
  return v;
}
template <int OFF> __device__ __forceinline__ void sts64o(unsigned addr, u64 v) {
  asm volatile("st.shared.u64 [%0+%1], %2;" ::"r"(addr), "n"(OFF), "l"(v) : "memory");
}
__device__ __forceinline__ void sts64(unsigned addr, u64 v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(addr), "l"(v) : "memory"); }

__device__ __forceinline__ unsigned lds32(unsigned addr) {
  unsigned v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

// mbarrier + 1-D bulk async copy (TMA engine, UBLKCP): one elected thread moves a whole contiguous
// tile global -> shared; the mbarrier counts the bytes that have landed
__device__ __forceinline__ void mbar_init(unsigned mbar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned mbar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned mbar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(mbar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(unsigned sdst, const void* gsrc, unsigned bytes, unsigned mbar) {
  asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(sdst), "l"(gsrc), "r"(bytes), "r"(mbar)
               : "memory");
}

// cp.async (LDGSTS): per-thread asynchronous global -> shared copy, zero-filled when !valid
__device__ __forceinline__ void cp_async8(unsigned sdst, const void* gsrc, bool valid) {
  int n = valid ? 8 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(sdst), "l"(gsrc), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async4(unsigned sdst, const void* gsrc, bool valid) {
  int n = valid ? 4 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(sdst), "l"(gsrc), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------------------------------------
// Float -> integer, one rule on every path (CVT, converting stores, store + reload through a storage dtype): NaN, +-inf
// and |x| >= 2^63 give INT64_MIN, anything else truncates toward zero, and a narrower integer dtype keeps the low bits
// of that int64.  This is what NumPy's astype(int64) gives on x86-64; a bare C cast would be PTX cvt.rzi, which clamps
// to the destination (+inf -> INT64_MAX, NaN -> 0, 3e9 -> int32 2147483647).
template <class T> __device__ __forceinline__ long long to_i64(T x) {
  if constexpr (std::is_floating_point<T>::value) return fabs(x) < T(9223372036854775808.0) ? (long long)x : (long long)0x8000000000000000ull;
  else return (long long)x;
}
// x as storage type S: integers through to_i64, floats by the C cast (int->float rn, f64->f32 rn)
template <class S, class T> __device__ __forceinline__ S to_storage(T x) {
  if constexpr (std::is_integral<S>::value) return (S)to_i64<T>(x);
  else return (S)x;
}

// ---------------------------------------------------------------------------------------------
// element loads / stores through explicit global-space instructions.
template <class S> __device__ __forceinline__ S ldg(const S* p) { return *p; }
template <> __device__ __forceinline__ double ldg<double>(const double* p) {
  double v;
  asm volatile("ld.global.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}
template <> __device__ __forceinline__ float ldg<float>(const float* p) {
  float v;
  asm volatile("ld.global.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
template <> __device__ __forceinline__ long long ldg<long long>(const long long* p) {
  long long v;
  asm volatile("ld.global.s64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
template <> __device__ __forceinline__ int ldg<int>(const int* p) {
  int v;
  asm volatile("ld.global.s32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
template <class S> __device__ __forceinline__ void stg(S* p, S v) { *p = v; }
template <> __device__ __forceinline__ void stg<double>(double* p, double v) { asm volatile("st.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }
template <> __device__ __forceinline__ void stg<float>(float* p, float v) { asm volatile("st.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }
template <> __device__ __forceinline__ void stg<long long>(long long* p, long long v) { asm volatile("st.global.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
template <> __device__ __forceinline__ void stg<int>(int* p, int v) { asm volatile("st.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

template <class T, class S, int V>
__device__ __forceinline__ void load_direct(const char* base, const long long (&off)[V], unsigned valid, T (&out)[V]) {
  const S* p = reinterpret_cast<const S*>(base);
  S tmp[V];
#pragma unroll
  for (int k = 0; k < V; ++k) tmp[k] = ((valid >> k) & 1u) ? ldg<S>(p + off[k]) : S(0);
#pragma unroll
  for (int k = 0; k < V; ++k) out[k] = (T)tmp[k];
}

template <class T> __device__ __noinline__ T load_narrow_one(const char* base, int dtype, long long off) {
  switch (dtype) {
    case RB200_BOOL:
    case RB200_U8: return (T) reinterpret_cast<const unsigned char*>(base)[off];
    case RB200_I8: return (T) reinterpret_cast<const signed char*>(base)[off];
    case RB200_I16: return (T) reinterpret_cast<const short*>(base)[off];
    case RB200_U16: return (T) reinterpret_cast<const unsigned short*>(base)[off];
    case RB200_U32: return (T) reinterpret_cast<const unsigned int*>(base)[off];
    default: return T(0);
  }
}

template <class T, int V>
__device__ __forceinline__ void load_view(const char* base, int dtype, const long long (&off)[V], unsigned valid, T (&out)[V]) {
  switch (dtype) {
    case RB200_F64: load_direct<T, double, V>(base, off, valid, out); break;
    case RB200_F32: load_direct<T, float, V>(base, off, valid, out); break;
    case RB200_I64: load_direct<T, long long, V>(base, off, valid, out); break;
    case RB200_I32: load_direct<T, int, V>(base, off, valid, out); break;
    default:  // narrow integer dtypes: off the hot path, out of line (static k: arrays stay in registers)
#pragma unroll
      for (int k = 0; k < V; ++k) out[k] = ((valid >> k) & 1u) ? load_narrow_one<T>(base, dtype, off[k]) : T(0);
  }
}

// staged element (natural layout: element e of the tile at slot + e*itemsize) -> compute class
template <class T> __device__ __forceinline__ T staged_load(unsigned slot_s, int e, int dtype) {
  switch (dtype) {
    case RB200_F64: return (T)__longlong_as_double((long long)lds64(slot_s + (unsigned)e * 8u));
    case RB200_I64: return (T)(long long)lds64(slot_s + (unsigned)e * 8u);
    case RB200_F32: return (T)__uint_as_float(lds32(slot_s + (unsigned)e * 4u));
    default: return (T)(int)lds32(slot_s + (unsigned)e * 4u);  // RB200_I32
  }
}

template <class T, class S, int V>
__device__ __forceinline__ void store_direct(char* base, const long long (&off)[V], unsigned mask, const T (&val)[V]) {
  S* p = reinterpret_cast<S*>(base);
#pragma unroll
  for (int k = 0; k < V; ++k)
    if ((mask >> k) & 1u) stg<S>(p + off[k], to_storage<S>(val[k]));
}

template <class T> __device__ __noinline__ void store_narrow_one(char* base, int dtype, long long off, T x) {
  switch (dtype) {
    case RB200_BOOL: reinterpret_cast<unsigned char*>(base)[off] = (x != T(0)) ? 1 : 0; break;
    case RB200_U8: reinterpret_cast<unsigned char*>(base)[off] = to_storage<unsigned char>(x); break;
    case RB200_I8: reinterpret_cast<signed char*>(base)[off] = to_storage<signed char>(x); break;
    case RB200_I16: reinterpret_cast<short*>(base)[off] = to_storage<short>(x); break;
    case RB200_U16: reinterpret_cast<unsigned short*>(base)[off] = to_storage<unsigned short>(x); break;
    case RB200_U32: reinterpret_cast<unsigned int*>(base)[off] = to_storage<unsigned int>(x); break;
    default: break;
  }
}

template <class T, int V>
__device__ __forceinline__ void store_view(char* base, int dtype, const long long (&off)[V], unsigned mask, const T (&val)[V]) {
  switch (dtype) {
    case RB200_F64: store_direct<T, double, V>(base, off, mask, val); break;
    case RB200_F32: store_direct<T, float, V>(base, off, mask, val); break;
    case RB200_I64: store_direct<T, long long, V>(base, off, mask, val); break;
    case RB200_I32: store_direct<T, int, V>(base, off, mask, val); break;
    default:
#pragma unroll
      for (int k = 0; k < V; ++k)
        if ((mask >> k) & 1u) store_narrow_one<T>(base, dtype, off[k], val[k]);
  }
}

// ---------------------------------------------------------------------------------------------
// fp64 sin/cos for V elements in lockstep (shared constants, no per-element branches):
// Cody-Waite reduction with a 3-part pi/2 and FMAs (j = rint(x*2/pi) by the 1.5*2^52 trick, exact
// for |x| < 2^31*pi/2), fdlibm kernel polynomials on [-pi/4, pi/4], quadrant select.  Against 200-bit
// references: at most 1.513 ulp on an H100 (tests/test_sincos_accuracy.py holds it to 1.55; the largest
// error among 3e8 arguments below 1e9, arange * 0.001 and uniform samples).  If any of a thread's V
// elements is 1e9 or more in magnitude, NaN or Inf, all V take the CUDA library routine (<= 2 ulp), so
// an element's result can differ by about 1 ulp with its neighbours.
// library routines out of line: their large-argument paths keep a table in local memory and would
// otherwise be inlined once per element into every trigonometric handler
static __device__ __noinline__ double2 sincos_lib(double x) {
  double2 r;
  sincos(x, &r.x, &r.y);
  return r;
}
static __device__ __noinline__ float2 sincosf_lib(float x) {
  float2 r;
  sincosf(x, &r.x, &r.y);
  return r;
}
template <int V> __device__ __forceinline__ void sincos_v(const double (&x)[V], double (&s)[V], double (&c)[V]) {
  bool big = false;
#pragma unroll
  for (int k = 0; k < V; ++k) big = big || !(fabs(x[k]) < 1.0e9);
  if (big) {
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const double2 r = sincos_lib(x[k]);
      s[k] = r.x;
      c[k] = r.y;
    }
    return;
  }
  const double TWO_OVER_PI = 0.6366197723675814, MAGIC = 6755399441055744.0;
  const double HI = 1.5707963267948966, MID = 6.123233995736766e-17, LO = -1.4973849048591698e-33;
  const double S1 = -1.66666666666666324348e-01, S2 = 8.33333333332248946124e-03, S3 = -1.98412698298579493134e-04,
               S4 = 2.75573137070700676789e-06, S5 = -2.50507602534068634195e-08, S6 = 1.58969099521155010221e-10;
  const double C1 = 4.16666666666666019037e-02, C2 = -1.38888888888741095749e-03, C3 = 2.48015872894767294178e-05,
               C4 = -2.75573143513906633035e-07, C5 = 2.08757232129817482790e-09, C6 = -1.13596475577881948265e-11;
#pragma unroll
  for (int k = 0; k < V; ++k) {
    const double t = fma(x[k], TWO_OVER_PI, MAGIC);
    const int q = __double2loint(t);
    const double j = t - MAGIC;
    double y = fma(-j, HI, x[k]);
    const double y2 = fma(-j, MID, y);
    y = fma(-j, LO, y2);
    const double z = y * y;
    double ps = fma(z, S6, S5);
    ps = fma(z, ps, S4);
    ps = fma(z, ps, S3);
    ps = fma(z, ps, S2);
    ps = fma(z, ps, S1);
    // sin(y) has the sign of y, and y that of y2 (|j * LO| < 1e-24, far below any nonzero |y2| for |x| < 1e9) - but
    // only y2 keeps x = -0 as -0: the last step adds -j * LO = +0 (j = +0, LO < 0), and so does the polynomial
    // (y * z * ps with ps < 0), and -0 + +0 is +0.  Taking the sign from y2 makes sin(-0) = -0 at the cost of one
    // LOP3, without a compare or a branch.
    const double sy = copysign(fma(y * z, ps, y), y2);
    double pc = fma(z, C6, C5);
    pc = fma(z, pc, C4);
    pc = fma(z, pc, C3);
    pc = fma(z, pc, C2);
    pc = fma(z, pc, C1);
    const double cy = fma(z, fma(z, pc, -0.5), 1.0);
    const double sn = (q & 1) ? cy : sy;
    const double cs = (q & 1) ? sy : cy;
    // sign flips: XOR the sign bit (bit 31 of the high word) with quadrant bit 1
    s[k] = __hiloint2double(__double2hiint(sn) ^ ((q & 2) << 30), __double2loint(sn));
    c[k] = __hiloint2double(__double2hiint(cs) ^ (((q + 1) & 2) << 30), __double2loint(cs));
  }
}
template <int V> __device__ __forceinline__ void sincos_v(const float (&x)[V], float (&s)[V], float (&c)[V]) {
#pragma unroll
  for (int k = 0; k < V; ++k) {
    const float2 r = sincosf_lib(x[k]);
    s[k] = r.x;
    c[k] = r.y;
  }
}

// ---------------------------------------------------------------------------------------------
// scalar op semantics

// Python floor division / modulo (what Numba emits for `//` and `%`).  A zero divisor gives 0 (no trap), and b = -1
// never reaches the hardware divide, whose INT64_MIN / -1 is undefined: the quotient wraps to INT64_MIN as NumPy's does.
__device__ __forceinline__ long long py_floordiv(long long a, long long b) {
  if (b == 0) return 0;
  if (b == -1) return (long long)(0ull - (u64)a);
  long long q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) --q;
  return q;
}
__device__ __forceinline__ long long py_mod(long long a, long long b) {
  if (b == 0 || b == -1) return 0;
  long long r = a % b;
  if (r != 0 && ((r < 0) != (b < 0))) r += b;
  return r;
}
template <class F> __device__ __forceinline__ F py_fmod(F a, F b) {
  F r = fmod(a, b);
  if (r != F(0)) {
    if ((b < F(0)) != (r < F(0))) r += b;
  } else {
    r = copysign(F(0), b);
  }
  return r;
}
template <class F> __device__ __forceinline__ F py_ffloordiv(F a, F b) {
  // CPython float_floor_div / Numba real_floordiv; a zero divisor gives a / b (+-inf, NaN for 0 / 0) as in Numba and
  // NumPy, where fmod(a, 0) = NaN would otherwise fall through to the result
  if (b == F(0)) return a / b;
  F mod = fmod(a, b);
  F div = (a - mod) / b;
  if (mod != F(0) && ((b < F(0)) != (mod < F(0)))) div -= F(1);
  if (div != F(0)) {
    F fl = floor(div);
    if (div - fl > F(0.5)) fl += F(1);
    return fl;
  }
  return copysign(F(0), a / b);
}

// x ** n for integer n: Numba's int_power_impl (exponentiation by squaring, r starts at 1)
template <class F> __device__ __forceinline__ F powi(F a, long long b) {
  bool invert = b < 0;
  u64 e = invert ? (u64)(-b) : (u64)b;
  if (e > 0x10000ull) return (F)pow((double)a, (double)b);
  F r = F(1);
  while (e != 0) {
    if (e & 1ull) r *= a;
    e >>= 1;
    a *= a;
  }
  return invert ? F(1) / r : r;
}
__device__ __forceinline__ long long ipowi(long long a, long long b) {
  if (b < 0) return (a == 1) ? 1 : ((a == -1) ? ((b & 1) ? -1 : 1) : 0);
  long long r = 1;
  u64 e = (u64)b;
  while (e != 0) {
    if (e & 1ull) r *= a;
    e >>= 1;
    a *= a;
  }
  return r;
}

// reduction combine in the accumulator class (raw bits).  MIN / MAX take a NaN from either side, so a NaN anywhere
// reaches the result wherever it sits in the tree (NumPy's min / max); the elementwise min / max binops do not.
template <class T> __device__ __forceinline__ T red_combine(int op, T a, T b) {
  switch (op) {
    case RB200_RED_ADD: return a + b;
    case RB200_RED_MUL: return a * b;
    case RB200_RED_MIN: return (b < a || b != b) ? b : a;
    default: return (b > a || b != b) ? b : a;
  }
}
__device__ __forceinline__ u64 red_combine_bits(int op, int ctype, u64 a, u64 b) {
  if (ctype == RB200_T_F64) return CT<double>::bits(red_combine<double>(op, CT<double>::get(a), CT<double>::get(b)));
  return CT<long long>::bits(red_combine<long long>(op, (long long)a, (long long)b));
}
__device__ __forceinline__ u64 red_identity_bits(int op, int ctype) {
  if (ctype == RB200_T_F64) {
    double d = (op == RB200_RED_ADD) ? 0.0 : (op == RB200_RED_MUL) ? 1.0 : (op == RB200_RED_MIN) ? INFINITY : -INFINITY;
    return CT<double>::bits(d);
  }
  long long i = (op == RB200_RED_ADD) ? 0ll : (op == RB200_RED_MUL) ? 1ll : (op == RB200_RED_MIN) ? 0x7fffffffffffffffll : (long long)0x8000000000000000ull;
  return (u64)i;
}

}  // namespace rb200
