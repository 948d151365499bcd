// rb200_philox.h — the value contract of RB200_OP_PHILOX (include/ramba_b200.h) as device code.  The general interpreter
// (rb200_interp.cuh) and the fill kernel (rb200_rng.cu) both evaluate draws through these functions only, so the two
// give the same bits for every element.
#pragma once
#include "../../include/ramba_b200.h"

namespace rb200 {

typedef unsigned long long rng_u64;

// Philox4x32-10 (Salmon, Moraes, Dror, Shaw, SC'11): ten rounds of two 32x32->64 multiplies and xors, key bumped by the
// Weyl constants between rounds.  Counter (c0, c1, c2, c3), key (k0, k1).
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, unsigned k0, unsigned k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// the block of draw `key` that element index `j` (already shifted to a block number) reads
__device__ __forceinline__ uint4 philox_block(rng_u64 j, rng_u64 key) {
  return philox4x32_10(make_uint4((unsigned)j, (unsigned)(j >> 32), 0u, 0u), (unsigned)key, (unsigned)(key >> 32));
}

__device__ __forceinline__ rng_u64 philox_half(uint4 w, int h) {
  return h ? ((rng_u64)w.w << 32 | w.z) : ((rng_u64)w.y << 32 | w.x);
}

// (x >> 11) * 2^-53: the 53-bit double in [0, 1)
__device__ __forceinline__ double philox_u01_64(rng_u64 x) { return __dmul_rn((double)(x >> 11), 0x1.0p-53); }
// (w >> 8) * 2^-24: the 24-bit float in [0, 1)
__device__ __forceinline__ float philox_u01_32(unsigned w) { return __fmul_rn((float)(w >> 8), 0x1.0p-24f); }
// mulhi64(x, n): x * n / 2^64 in [0, n)
__device__ __forceinline__ long long philox_bounded(rng_u64 x, rng_u64 n) { return (long long)__umul64hi(x, n); }

// Box-Muller pair of one block, every step rounded on its own.  Out of line, so that both kernels run the very same
// instructions (the interpreter keeps one half of the pair, the fill kernel both).
static __device__ __noinline__ double2 philox_normal_pair(uint4 w) {
  const double u1 = __dsub_rn(1.0, philox_u01_64(philox_half(w, 0)));  // (0, 1]: log is finite
  const double u2 = philox_u01_64(philox_half(w, 1));
  const double r = sqrt(__dmul_rn(-2.0, log(u1)));
  const double t = __dmul_rn(6.283185307179586, u2);
  return make_double2(__dmul_rn(r, cos(t)), __dmul_rn(r, sin(t)));
}

// element `i` of draw `key` in output form `form` (bound `n` for the integer form), as the raw 64-bit value of the
// form's compute class (double bits, float bits in the low word, int64)
static __device__ __noinline__ rng_u64 philox_element_bits(long long i, rng_u64 key, rng_u64 n, unsigned form) {
  const rng_u64 u = (rng_u64)i;
  switch (form) {
    case RB200_PHILOX_UNIFORM32: {
      const uint4 w = philox_block(u >> 2, key);
      const unsigned k = (unsigned)u & 3u;
      const unsigned x = k == 0 ? w.x : k == 1 ? w.y : k == 2 ? w.z : w.w;
      return (rng_u64)__float_as_uint(philox_u01_32(x));
    }
    case RB200_PHILOX_NORMAL64: {
      const double2 z = philox_normal_pair(philox_block(u >> 1, key));
      return (rng_u64)__double_as_longlong((u & 1) ? z.y : z.x);
    }
    case RB200_PHILOX_INTEGER: return (rng_u64)philox_bounded(philox_half(philox_block(u >> 1, key), (int)(u & 1)), n);
    default: return (rng_u64)__double_as_longlong(philox_u01_64(philox_half(philox_block(u >> 1, key), (int)(u & 1))));
  }
}

}  // namespace rb200
