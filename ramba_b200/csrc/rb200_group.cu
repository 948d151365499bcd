// rb200_group.cu — grouped reduction along one axis on sm_90a: out[o, g, i] = op over the members t of group g of src[o, t, i].
//
// What it stands for in the reference: RambaGroupby's aggregations (ramba/ramba.py:10185-10643), which run
// sreduce_index over Python callables on the workers.  Here the host turns the labels into a CSR table once (offsets,
// and the positions of every group in ascending order) and one launch reads every source element once.
//
// Fold order (the same for every form, so that the bits depend only on the view's shape, G and the labels): the grouped
// axis is cut into S chunks of C positions (the plan picks C); the members of a group inside one chunk are combined in
// ascending order starting from the op's identity, and the S chunk partials of an output are combined in chunk order,
// again starting from the identity.  No atomics.
//   * row form (the grouped axis has unit stride and nothing follows it): one CTA per row, or K CTAs per row when there
//     are too few rows to fill the GPU.  A CTA stages its part of the row in shared memory 32 KB at a time and every thread
//     walks the members of up to four (chunk, group) items; when a row fits one CTA and there are few groups, the row is
//     cut into several chunks so that more threads have work, and their partials are folded in shared memory.
//   * column form (the dims after the axis collapse to one contiguous run of >= 32 elements) and general form (any other
//     view): one thread per kept element (o, i) and group; loads of neighbouring threads are neighbouring elements in the
//     column form.
//   * split (any form): partials go to `scratch` as part[s * N + j] (N outputs) and one more kernel folds them.
// Floating-point sources accumulate in float64, integers in int64 with wrap-around; products, sums and the squared
// deviations are rounded separately (no FMA contraction).
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>
#include <type_traits>

#include "rb200_group.h"

namespace rb200 {

constexpr int kGThreads = 256;
constexpr int kKPT = 4;                   // (chunk, group) items per thread in the row form
constexpr int kRowMaxItems = kGThreads * kKPT;
constexpr int kTileBytes = 32768;         // row form: shared-memory tile of the row
constexpr long long kPlanSms = 132;       // H100 SXM: the plan (and so the fold order) does not depend on the device
constexpr long long kTargetCtas = 4 * kPlanSms;
constexpr long long kMinChunk = 1024;     // positions per chunk when the axis is split across CTAs
constexpr long long kMaxSplit = 1024;

template <class TS> struct IsFloat { static constexpr bool value = std::is_floating_point<TS>::value; };

template <class TS, int OP> struct GAcc {
  using A = typename std::conditional<IsFloat<TS>::value || OP == RB200_GROUP_SQDEV, double, long long>::type;
};

template <class A, int OP> __device__ __forceinline__ A g_identity() {
  if (OP == RB200_GROUP_PROD) return A(1);
  if (OP == RB200_GROUP_MIN) return std::is_same<A, double>::value ? A(INFINITY) : A(0x7fffffffffffffffll);
  if (OP == RB200_GROUP_MAX) return std::is_same<A, double>::value ? A(-INFINITY) : A((long long)0x8000000000000000ull);
  return A(0);
}

__device__ __forceinline__ double g_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ long long g_add(long long a, long long b) { return (long long)((unsigned long long)a + (unsigned long long)b); }
__device__ __forceinline__ double g_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ long long g_mul(long long a, long long b) { return (long long)((unsigned long long)a * (unsigned long long)b); }

// partial (op) partial
template <class A, int OP> __device__ __forceinline__ A g_combine(A a, A b) {
  if (OP == RB200_GROUP_PROD) return g_mul(a, b);
  if (OP == RB200_GROUP_MIN) return (b < a) ? b : a;
  if (OP == RB200_GROUP_MAX) return (b > a) ? b : a;
  return g_add(a, b);
}

// accumulator (op) one source element
template <class TS, int OP, class A> __device__ __forceinline__ A g_step(A acc, TS x, double c) {
  if constexpr (OP == RB200_GROUP_SQDEV) {
    const double d = __dsub_rn((double)x, c);
    return __dadd_rn(acc, __dmul_rn(d, d));
  } else if constexpr (OP == RB200_GROUP_NANCOUNT) {
    if constexpr (IsFloat<TS>::value) return x != x ? acc : g_add(acc, A(1));
    else return g_add(acc, A(1));
  } else if constexpr (OP == RB200_GROUP_NANSUM) {
    if constexpr (IsFloat<TS>::value) return x != x ? acc : g_add(acc, (A)x);
    else return g_add(acc, (A)x);
  } else {
    return g_combine<A, OP>(acc, (A)x);
  }
}

// first index in members[lo, hi) whose position is >= key (members ascending there)
__device__ __forceinline__ long long lower_bound(const long long* __restrict__ m, long long lo, long long hi, long long key) {
  while (lo < hi) {
    const long long mid = lo + ((hi - lo) >> 1);
    if (m[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// element offset of kept element k (C order over the kept dims)
__device__ __forceinline__ long long kept_offset(const GroupPlan& P, long long k) {
  long long off = 0;
#pragma unroll
  for (int d = RB200_MAX_DIMS - 2; d >= 0; --d) {
    if (d < P.nk) {
      const long long q = k / P.kshape[d];
      off += (k - q * P.kshape[d]) * P.kstride[d];
      k = q;
    }
  }
  return off;
}

template <class TS, int OP>
__global__ void __launch_bounds__(kGThreads, 1)
    group_row_kernel(const __grid_constant__ GroupPlan P, const long long* __restrict__ offsets, const long long* __restrict__ members,
                     const double* __restrict__ center, typename GAcc<TS, OP>::A* __restrict__ out, typename GAcc<TS, OP>::A* __restrict__ part) {
  using A = typename GAcc<TS, OP>::A;
  constexpr int kCap = kTileBytes / (int)sizeof(TS);
  extern __shared__ __align__(16) unsigned char g_smem[];
  TS* tile = reinterpret_cast<TS*>(g_smem);
  A* pf = reinterpret_cast<A*>(g_smem + kTileBytes);
  const long long o = blockIdx.x / P.K;
  const int kc = (int)(blockIdx.x - o * P.K);
  const TS* __restrict__ row = reinterpret_cast<const TS*>(P.base) + kept_offset(P, o);
  const long long T0 = (long long)kc * P.ncl * P.C;
  const long long T1 = min(P.L, T0 + (long long)P.ncl * P.C);
  const int n_items = P.G * P.ncl;
  A acc[kKPT];
  long long cur[kKPT], end[kKPT];
  double cen[kKPT];
#pragma unroll
  for (int q = 0; q < kKPT; ++q) {
    const int j = threadIdx.x + q * kGThreads;
    acc[q] = g_identity<A, OP>();
    cur[q] = end[q] = 0;
    cen[q] = 0.0;
    if (j < n_items) {
      const int c = j / P.G, g = j - c * P.G;
      const long long lo = T0 + (long long)c * P.C, hi = min(lo + P.C, T1);
      const long long b = offsets[g], e = offsets[g + 1];
      cur[q] = P.S == 1 ? b : lower_bound(members, b, e, lo);
      end[q] = P.S == 1 ? e : lower_bound(members, cur[q], e, hi);
      if (OP == RB200_GROUP_SQDEV) cen[q] = center[o * P.G + g];
    }
  }
  for (long long p0 = T0; p0 < T1; p0 += kCap) {
    const int n = (int)min((long long)kCap, T1 - p0);
    __syncthreads();
#pragma unroll 4
    for (int j = threadIdx.x; j < n; j += kGThreads) tile[j] = __ldcs(row + p0 + j);
    __syncthreads();
    const long long pend = p0 + n;
#pragma unroll
    for (int q = 0; q < kKPT; ++q) {
      while (cur[q] < end[q]) {  // four member positions at a time; they ascend, so the ones in this tile are a prefix
        long long t[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) t[u] = cur[q] + u < end[q] ? members[cur[q] + u] : 0x7fffffffffffffffll;
        int nb = 0;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (t[u] < pend) {
            acc[q] = g_step<TS, OP>(acc[q], tile[t[u] - p0], cen[q]);
            ++nb;
          }
        }
        cur[q] += nb;
        if (nb < 4) break;
      }
    }
  }
  if (P.K == 1) {  // the whole row: fold the chunk partials in chunk order here
#pragma unroll
    for (int q = 0; q < kKPT; ++q) {
      const int j = threadIdx.x + q * kGThreads;
      if (j < n_items) pf[j] = acc[q];
    }
    __syncthreads();
    for (int g = threadIdx.x; g < P.G; g += kGThreads) {
      A r = g_identity<A, OP>();
      for (int c = 0; c < P.ncl; ++c) r = g_combine<A, OP>(r, pf[c * P.G + g]);
      out[o * P.G + g] = r;
    }
  } else {  // one chunk per CTA (ncl == 1): item j is group j
    const long long N = P.O * P.G;
#pragma unroll
    for (int q = 0; q < kKPT; ++q) {
      const int j = threadIdx.x + q * kGThreads;
      if (j < n_items) part[(long long)kc * N + o * P.G + j] = acc[q];
    }
  }
}

template <class TS, int OP>
__global__ void __launch_bounds__(kGThreads, 1)
    group_kept_kernel(const __grid_constant__ GroupPlan P, const long long* __restrict__ offsets, const long long* __restrict__ members,
                      const double* __restrict__ center, typename GAcc<TS, OP>::A* __restrict__ out, typename GAcc<TS, OP>::A* __restrict__ part) {
  using A = typename GAcc<TS, OP>::A;
  const long long tile = blockIdx.x / P.S;
  const int s = (int)(blockIdx.x - tile * P.S);
  const long long k = tile * kGThreads + threadIdx.x;
  if (k >= P.nkept) return;
  const TS* __restrict__ src = reinterpret_cast<const TS*>(P.base) + kept_offset(P, k);
  const long long o = k / P.I, i = k - o * P.I;
  const long long lo = (long long)s * P.C, hi = min(lo + P.C, P.L);
  const long long N = P.nkept * P.G;
  for (int g = blockIdx.y; g < P.G; g += gridDim.y) {
    const long long b = offsets[g], e = offsets[g + 1];
    long long cur = P.S == 1 ? b : lower_bound(members, b, e, lo);
    const long long end = P.S == 1 ? e : lower_bound(members, cur, e, hi);
    const long long oi = (o * P.G + g) * P.I + i;
    const double c = OP == RB200_GROUP_SQDEV ? center[oi] : 0.0;
    A acc = g_identity<A, OP>();
    for (; cur + 4 <= end; cur += 4) {
      long long t[4];
      TS x[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) t[u] = members[cur + u];
#pragma unroll
      for (int u = 0; u < 4; ++u) x[u] = __ldcs(src + t[u] * P.sa);
#pragma unroll
      for (int u = 0; u < 4; ++u) acc = g_step<TS, OP>(acc, x[u], c);
    }
    for (; cur < end; ++cur) acc = g_step<TS, OP>(acc, __ldcs(src + members[cur] * P.sa), c);
    if (P.S == 1) out[oi] = g_combine<A, OP>(g_identity<A, OP>(), acc);
    else part[(long long)s * N + oi] = acc;
  }
}

// out[j] = identity (op) part[0*N + j] (op) part[1*N + j] ... in chunk order
template <class A, int OP> __global__ void __launch_bounds__(kGThreads) group_fold_kernel(const A* __restrict__ part, A* __restrict__ out, long long N, int S) {
  for (long long j = (long long)blockIdx.x * kGThreads + threadIdx.x; j < N; j += (long long)gridDim.x * kGThreads) {
    A r = g_identity<A, OP>();
    int s = 0;
    for (; s + 8 <= S; s += 8) {
      A v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = part[(long long)(s + u) * N + j];
#pragma unroll
      for (int u = 0; u < 8; ++u) r = g_combine<A, OP>(r, v[u]);
    }
    for (; s < S; ++s) r = g_combine<A, OP>(r, part[(long long)s * N + j]);
    out[j] = r;
  }
}

// ---- host: plan and dispatch --------------------------------------------------------------------------------------------
static long long cdiv(long long a, long long b) { return (a + b - 1) / b; }

const char* group_form_name(int form) { return form == GFORM_ROW ? "row" : form == GFORM_COLUMN ? "column" : "general"; }

void make_group_plan(const rb200_index_view& v, int axis, int n_groups, GroupPlan* P) {
  GroupPlan& p = *P;
  p.base = (const char*)v.base;
  p.elem_bytes = v.elem_bytes;
  p.G = n_groups;
  p.L = v.shape[axis];
  p.sa = v.stride[axis];
  p.nk = 0;
  p.O = p.I = 1;
  int n_outer = 0;
  for (int side = 0; side < 2; ++side) {
    const int first = p.nk, d0 = side == 0 ? 0 : axis + 1, d1 = side == 0 ? axis : v.ndim;
    for (int d = d0; d < d1; ++d) {
      (side == 0 ? p.O : p.I) *= v.shape[d];
      if (v.shape[d] == 1) continue;
      if (p.nk > first && p.kstride[p.nk - 1] == v.stride[d] * v.shape[d]) {  // contiguous with the previous kept dim
        p.kshape[p.nk - 1] *= v.shape[d];
        p.kstride[p.nk - 1] = v.stride[d];
        continue;
      }
      p.kshape[p.nk] = v.shape[d];
      p.kstride[p.nk] = v.stride[d];
      ++p.nk;
    }
    if (side == 0) n_outer = p.nk;
  }
  p.nkept = p.O * p.I;
  const int n_inner = p.nk - n_outer;
  if (p.I == 1 && p.sa == 1 && n_groups <= kRowMaxItems) p.form = GFORM_ROW;
  else if (n_inner == 1 && p.kstride[p.nk - 1] == 1 && p.kshape[p.nk - 1] >= 32) p.form = GFORM_COLUMN;
  else p.form = GFORM_GENERAL;
  const long long L = p.L;
  p.K = 1;
  p.ncl = 1;
  if (p.form == GFORM_ROW) {
    long long K = 1;
    if (p.O < kTargetCtas && L >= 2 * kMinChunk) K = std::min(cdiv(kTargetCtas, std::max(p.O, 1ll)), L / kMinChunk);
    if (K <= 1) {  // one CTA per row; few groups: several chunks so that more threads walk
      long long ncl = std::min(std::min(64ll, cdiv(kGThreads, n_groups)), std::max(L, 1ll));
      p.C = std::max(cdiv(L, ncl), 1ll);
      p.ncl = (int)std::max(cdiv(L, p.C), 1ll);
      p.S = p.ncl;
    } else {
      p.C = cdiv(L, K);
      p.K = (int)cdiv(L, p.C);
      p.S = p.K;
    }
    p.ctas = p.O * p.K;
  } else {
    const long long base = cdiv(p.nkept, kGThreads) * n_groups;
    long long S = 1;
    if (base < kTargetCtas && L >= 2 * kMinChunk) S = std::min(std::min(cdiv(kTargetCtas, std::max(base, 1ll)), L / kMinChunk), kMaxSplit);
    p.C = std::max(cdiv(L, S), 1ll);
    p.S = (int)std::max(cdiv(L, p.C), 1ll);
    p.ctas = cdiv(p.nkept, kGThreads) * p.S * std::min(n_groups, 65535);
  }
  const bool split = p.form == GFORM_ROW ? p.K > 1 : p.S > 1;
  p.scratch_bytes = split ? (long long)p.S * p.nkept * n_groups * 8 : 0;
}

template <class TS, int OP>
static cudaError_t launch_t(const GroupPlan& P, const long long* offsets, const long long* members, const double* center, void* out, void* scratch,
                            cudaStream_t s) {
  using A = typename GAcc<TS, OP>::A;
  A* dst = (A*)out;
  A* part = (A*)scratch;
  if (P.form == GFORM_ROW) {
    const int smem = kTileBytes + kRowMaxItems * 8;
    group_row_kernel<TS, OP><<<(unsigned)P.ctas, kGThreads, smem, s>>>(P, offsets, members, center, dst, part);
  } else {
    const dim3 grid((unsigned)(cdiv(P.nkept, kGThreads) * P.S), (unsigned)std::min(P.G, 65535));
    group_kept_kernel<TS, OP><<<grid, kGThreads, 0, s>>>(P, offsets, members, center, dst, part);
  }
  if (P.scratch_bytes) {
    const long long N = P.nkept * P.G;
    const long long blocks = std::min(cdiv(N, kGThreads), kPlanSms * 8);
    group_fold_kernel<A, OP><<<(unsigned)blocks, kGThreads, 0, s>>>(part, dst, N, P.S);
  }
  return cudaGetLastError();
}

template <class TS>
static cudaError_t launch_op(const GroupPlan& P, int op, const long long* offsets, const long long* members, const double* center, void* out, void* scratch,
                             cudaStream_t s) {
  switch (op) {
    case RB200_GROUP_SUM: return launch_t<TS, RB200_GROUP_SUM>(P, offsets, members, center, out, scratch, s);
    case RB200_GROUP_PROD: return launch_t<TS, RB200_GROUP_PROD>(P, offsets, members, center, out, scratch, s);
    case RB200_GROUP_MIN: return launch_t<TS, RB200_GROUP_MIN>(P, offsets, members, center, out, scratch, s);
    case RB200_GROUP_MAX: return launch_t<TS, RB200_GROUP_MAX>(P, offsets, members, center, out, scratch, s);
    case RB200_GROUP_NANSUM: return launch_t<TS, RB200_GROUP_NANSUM>(P, offsets, members, center, out, scratch, s);
    case RB200_GROUP_NANCOUNT: return launch_t<TS, RB200_GROUP_NANCOUNT>(P, offsets, members, center, out, scratch, s);
    default: return launch_t<TS, RB200_GROUP_SQDEV>(P, offsets, members, center, out, scratch, s);
  }
}

cudaError_t launch_group(const GroupPlan& P, int src_dtype, int op, const long long* offsets, const long long* members, const double* center,
                         void* out, void* scratch, cudaStream_t s) {
  if (P.nkept == 0) return cudaSuccess;
  switch (src_dtype) {
    case RB200_F64: return launch_op<double>(P, op, offsets, members, center, out, scratch, s);
    case RB200_F32: return launch_op<float>(P, op, offsets, members, center, out, scratch, s);
    case RB200_I64: return launch_op<long long>(P, op, offsets, members, center, out, scratch, s);
    default: return launch_op<int>(P, op, offsets, members, center, out, scratch, s);
  }
}

}  // namespace rb200
