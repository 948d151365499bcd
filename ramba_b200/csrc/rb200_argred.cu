// rb200_argred.cu — first-occurrence index reductions on sm_90a: argmax, argmin, nanargmax and nanargmin of a strided
// view, over all its axes or along one, emitting global indices.
//
// Every element becomes an int64 order key (include/ramba_b200.h states the rule), so that all four ops become "largest
// key, then smallest index".  That pair is a total order, so the answer does not depend on the grid, the split or the
// fold order: any launch shape gives the same index.  No atomics.
//   * global form (all axes): each CTA walks one contiguous chunk of the view's C-order positions (16-byte vector loads
//     when the view is one unit-stride run) and leaves one (key, index) partial; a fold kernel finishes.
//   * row form (unit-stride axis, nothing kept after it): one warp per output row, vector loads across the warp.
//   * column form (the kept dims after the axis merge into one unit-stride run of >= 32) and general form (any other
//     view): one thread per output; in the column form neighbouring threads load neighbouring elements.
//   * split: an axis form whose outputs cannot fill the GPU cuts the axis into S chunks; the partials go to scratch as
//     part[s * n_out + j] and the same fold kernel finishes.
// Inside one thread the positions are visited in ascending order, so a tie keeps the first; positions are turned into
// global indices once per thread (the local C order of a box of the global array is ascending in the global index).
#include <cuda_runtime.h>

#include <algorithm>
#include <type_traits>

#include "rb200_argred.h"

namespace rb200 {

constexpr int kAThreads = 256;
constexpr int kAWarps = kAThreads / 32;
constexpr long long kArgPlanSms = 132;  // H100 SXM: the plan does not depend on the device
constexpr long long kArgTargetCtas = 8 * kArgPlanSms;
constexpr long long kArgMinChunk = 1024;  // positions per chunk when an axis is split
constexpr long long kArgMaxSplit = 1024;
constexpr long long kArgChunkAlign = 64;  // chunk starts stay 16-byte aligned when the view's start is
constexpr long long kNoIndex = 0x7fffffffffffffffll;
constexpr long long kKeyMin = (long long)0x8000000000000000ull;

template <class TS> struct ArgIsFloat { static constexpr bool value = std::is_floating_point<TS>::value; };

__device__ __forceinline__ long long arg_bits(double x) { return __double_as_longlong(x); }
__device__ __forceinline__ long long arg_bits(float x) { return (long long)__float_as_int(x); }  // sign-extended

// the order key of one element; *ok is false for a NaN of a nan variant (no candidate)
template <class TS, int OP> __device__ __forceinline__ long long arg_key(TS x, bool* ok) {
  long long k;
  *ok = true;
  if constexpr (ArgIsFloat<TS>::value) {
    long long b = arg_bits(x);
    if (x == TS(0)) b = 0;  // -0.0 == 0.0: one key
    k = b >= 0 ? b : b ^ 0x7fffffffffffffffll;
    if (x != x) {
      *ok = OP == RB200_ARG_MAX || OP == RB200_ARG_MIN;
      k = OP == RB200_ARG_MIN ? kKeyMin : kNoIndex;  // after argmin's flip a NaN is the largest key too
    }
  } else {
    k = (long long)x;
  }
  return (OP == RB200_ARG_MIN || OP == RB200_ARG_NANMIN) ? ~k : k;
}

// the best (largest key) position a thread has seen; positions arrive ascending, so a tie keeps the first
struct ArgBest {
  long long k, t;
};

template <class TS, int OP> __device__ __forceinline__ void arg_take(ArgBest& b, TS x, long long t) {
  bool ok;
  const long long k = arg_key<TS, OP>(x, &ok);
  if (ok && (k > b.k || b.t < 0)) {
    b.k = k;
    b.t = t;
  }
}

// (key, index) pairs: the larger key, then the smaller index
__device__ __forceinline__ void arg_merge(long long& k, long long& i, long long k2, long long i2) {
  if (k2 > k || (k2 == k && i2 < i)) {
    k = k2;
    i = i2;
  }
}

__device__ __forceinline__ void arg_warp_merge(long long& k, long long& i) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) arg_merge(k, i, __shfl_xor_sync(0xffffffffu, k, off), __shfl_xor_sync(0xffffffffu, i, off));
}

// element offset (or flat index) of position t of a C-order walk over nd dims
__device__ __forceinline__ long long arg_decode(const long long* shape, const long long* st, int nd, long long t) {
  long long off = 0;
#pragma unroll
  for (int d = RB200_MAX_DIMS - 1; d >= 0; --d) {
    if (d < nd) {
      const long long q = t / shape[d];
      off += (t - q * shape[d]) * st[d];
      t = q;
    }
  }
  return off;
}

template <class TS> struct ArgVec;
template <> struct ArgVec<double> { using T = double2; static constexpr int n = 2; };
template <> struct ArgVec<float> { using T = float4; static constexpr int n = 4; };
template <> struct ArgVec<long long> { using T = longlong2; static constexpr int n = 2; };
template <> struct ArgVec<int> { using T = int4; static constexpr int n = 4; };

template <class V> __device__ __forceinline__ auto arg_lane(const V& v, int u) -> decltype(v.x) {
  if constexpr (sizeof(v) / sizeof(v.x) == 2) return u == 0 ? v.x : v.y;
  else return u == 0 ? v.x : u == 1 ? v.y : u == 2 ? v.z : v.w;
}

// positions tbase + [0, n) of the unit-stride run p[0, n), walked by NL lanes: scalar head up to 16-byte alignment,
// four 16-byte vectors in flight per lane, scalar tail
template <class TS, int OP, int NL> __device__ __forceinline__ void arg_scan_run(const TS* __restrict__ p, long long n, int lane, long long tbase, ArgBest& b) {
  using VT = typename ArgVec<TS>::T;
  constexpr int V = ArgVec<TS>::n;
  const long long head = min(n, (long long)(((16 - ((unsigned long long)p & 15)) & 15) / sizeof(TS)));
  for (long long j = lane; j < head; j += NL) arg_take<TS, OP>(b, __ldcs(p + j), tbase + j);
  const VT* __restrict__ q = reinterpret_cast<const VT*>(p + head);
  const long long nv = (n - head) / V;
  const long long t0 = tbase + head;
  long long j = lane;
  for (; j + 3 * NL < nv; j += 4 * NL) {
    VT v[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) v[r] = __ldcs(q + j + r * NL);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int u = 0; u < V; ++u) arg_take<TS, OP>(b, (TS)arg_lane(v[r], u), t0 + (j + r * NL) * V + u);
  }
  for (; j < nv; j += NL) {
    const VT v = __ldcs(q + j);
#pragma unroll
    for (int u = 0; u < V; ++u) arg_take<TS, OP>(b, (TS)arg_lane(v, u), t0 + j * V + u);
  }
  for (long long t = head + nv * V + lane; t < n; t += NL) arg_take<TS, OP>(b, __ldcs(p + t), tbase + t);
}

// the CTA's best pair into (k, i) of thread 0
__device__ __forceinline__ void arg_cta_merge(long long& k, long long& i) {
  __shared__ long long sk[kAWarps], si[kAWarps];
  arg_warp_merge(k, i);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    sk[w] = k;
    si[w] = i;
  }
  __syncthreads();
  if (w == 0) {
    k = lane < kAWarps ? sk[lane] : kKeyMin;
    i = lane < kAWarps ? si[lane] : kNoIndex;
    arg_warp_merge(k, i);
  }
}

__device__ __forceinline__ void arg_write(const ArgPlan& P, long long j, int s, long long k, long long i, long long* out_idx, long long* out_key,
                                          longlong2* part) {
  if (P.S == 1) {
    out_idx[j] = i;
    out_key[j] = k;
  } else {
    part[(long long)s * P.n_out + j] = make_longlong2(k, i);
  }
}

template <class TS, int OP>
__global__ void __launch_bounds__(kAThreads) arg_global_kernel(const __grid_constant__ ArgPlan P, long long* __restrict__ out_idx,
                                                               long long* __restrict__ out_key, longlong2* __restrict__ part) {
  const TS* __restrict__ src = reinterpret_cast<const TS*>(P.base);
  const long long lo = (long long)blockIdx.x * P.C, hi = min(lo + P.C, P.L);
  ArgBest b{kKeyMin, -1};
  if (P.nd == 1 && P.stride[0] == 1) {
    if (lo < hi) arg_scan_run<TS, OP, kAThreads>(src + lo, hi - lo, threadIdx.x, lo, b);
  } else if (P.nd == 1) {
    for (long long t = lo + threadIdx.x; t < hi; t += kAThreads) arg_take<TS, OP>(b, __ldcs(src + t * P.stride[0]), t);
  } else {
    for (long long t = lo + threadIdx.x; t < hi; t += kAThreads) arg_take<TS, OP>(b, __ldcs(src + arg_decode(P.shape, P.stride, P.nd, t)), t);
  }
  long long k = b.k, i = b.t < 0 ? kNoIndex : P.g0 + arg_decode(P.shape, P.gstride, P.nd, b.t);
  arg_cta_merge(k, i);
  if (threadIdx.x == 0) arg_write(P, 0, blockIdx.x, k, i, out_idx, out_key, part);
}

template <class TS, int OP>
__global__ void __launch_bounds__(kAThreads) arg_row_kernel(const __grid_constant__ ArgPlan P, long long* __restrict__ out_idx,
                                                            long long* __restrict__ out_key, longlong2* __restrict__ part) {
  const long long gw = (long long)blockIdx.x * kAWarps + (threadIdx.x >> 5);
  if (gw >= P.n_out * P.S) return;  // (a whole warp)
  const int lane = threadIdx.x & 31;
  const long long o = gw / P.S;
  const int s = (int)(gw - o * P.S);
  const TS* __restrict__ row = reinterpret_cast<const TS*>(P.base) + arg_decode(P.shape, P.stride, P.nd, o);
  const long long lo = (long long)s * P.C, hi = min(lo + P.C, P.L);
  ArgBest b{kKeyMin, -1};
  if (lo < hi) arg_scan_run<TS, OP, 32>(row + lo, hi - lo, lane, lo, b);
  long long k = b.k, i = b.t < 0 ? kNoIndex : P.g0 + b.t;
  arg_warp_merge(k, i);
  if (lane == 0) arg_write(P, o, s, k, i, out_idx, out_key, part);
}

template <class TS, int OP>
__global__ void __launch_bounds__(kAThreads) arg_kept_kernel(const __grid_constant__ ArgPlan P, long long* __restrict__ out_idx,
                                                             long long* __restrict__ out_key, longlong2* __restrict__ part) {
  const long long tile = blockIdx.x / P.S;
  const int s = (int)(blockIdx.x - tile * P.S);
  const long long j = tile * kAThreads + threadIdx.x;
  if (j >= P.n_out) return;
  const TS* __restrict__ src = reinterpret_cast<const TS*>(P.base) + arg_decode(P.shape, P.stride, P.nd, j);
  const long long lo = (long long)s * P.C, hi = min(lo + P.C, P.L);
  ArgBest b{kKeyMin, -1};
  long long t = lo;
  for (; t + 8 <= hi; t += 8) {
    TS x[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) x[u] = __ldcs(src + (t + u) * P.sa);
#pragma unroll
    for (int u = 0; u < 8; ++u) arg_take<TS, OP>(b, x[u], t + u);
  }
  for (; t < hi; ++t) arg_take<TS, OP>(b, __ldcs(src + t * P.sa), t);
  arg_write(P, j, s, b.k, b.t < 0 ? kNoIndex : P.g0 + b.t, out_idx, out_key, part);
}

// one warp per output: the best of its S partials
__global__ void __launch_bounds__(kAThreads) arg_fold_kernel(const longlong2* __restrict__ part, long long* __restrict__ out_idx,
                                                             long long* __restrict__ out_key, long long n_out, int S) {
  const long long j = (long long)blockIdx.x * kAWarps + (threadIdx.x >> 5);
  if (j >= n_out) return;
  const int lane = threadIdx.x & 31;
  long long k = kKeyMin, i = kNoIndex;
  for (int s = lane; s < S; s += 32) {
    const longlong2 v = part[(long long)s * n_out + j];
    arg_merge(k, i, v.x, v.y);
  }
  arg_warp_merge(k, i);
  if (lane == 0) {
    out_idx[j] = i;
    out_key[j] = k;
  }
}

// ---- host: plan and dispatch --------------------------------------------------------------------------------------------
static long long arg_cdiv(long long a, long long b) { return (a + b - 1) / b; }

const char* arg_form_name(int form) {
  return form == AFORM_GLOBAL ? "global" : form == AFORM_ROW ? "row" : form == AFORM_COLUMN ? "column" : "general";
}

void make_arg_plan(const rb200_index_view& v, int axis, ArgPlan* P) {
  ArgPlan& p = *P;
  p.base = (const char*)v.base;
  p.nd = 0;
  p.g0 = 0;
  p.sa = 0;
  if (axis == RB200_ARG_ALL_AXES) {
    p.form = AFORM_GLOBAL;
    p.L = 1;
    for (int d = 0; d < v.ndim; ++d) {
      p.L *= v.shape[d];
      if (v.shape[d] == 1) continue;
      p.shape[p.nd] = v.shape[d];
      p.stride[p.nd] = v.stride[d];
      p.gstride[p.nd] = 0;
      ++p.nd;
    }
    if (p.nd == 0) {  // a single element
      p.shape[0] = 1;
      p.stride[0] = 1;
      p.gstride[0] = 0;
      p.nd = 1;
    }
    p.n_out = 1;
    const long long ctas = std::max(1ll, std::min(kArgTargetCtas, arg_cdiv(p.L, kAThreads * 16)));
    p.C = std::max(arg_cdiv(arg_cdiv(p.L, ctas), kArgChunkAlign) * kArgChunkAlign, kArgChunkAlign);
    p.S = (int)std::max(arg_cdiv(p.L, p.C), 1ll);
    p.ctas = p.S;
  } else {
    p.L = v.shape[axis];
    p.sa = v.stride[axis];
    long long O = 1, I = 1;
    int n_outer = 0;
    for (int side = 0; side < 2; ++side) {
      const int first = p.nd, d0 = side == 0 ? 0 : axis + 1, d1 = side == 0 ? axis : v.ndim;
      for (int d = d0; d < d1; ++d) {
        (side == 0 ? O : I) *= v.shape[d];
        if (v.shape[d] == 1) continue;
        if (p.nd > first && p.stride[p.nd - 1] == v.stride[d] * v.shape[d]) {  // contiguous with the previous kept dim
          p.shape[p.nd - 1] *= v.shape[d];
          p.stride[p.nd - 1] = v.stride[d];
          continue;
        }
        p.shape[p.nd] = v.shape[d];
        p.stride[p.nd] = v.stride[d];
        ++p.nd;
      }
      if (side == 0) n_outer = p.nd;
    }
    p.n_out = O * I;
    const int n_inner = p.nd - n_outer;
    if (I == 1 && p.sa == 1) p.form = AFORM_ROW;
    else if (n_inner == 1 && p.stride[p.nd - 1] == 1 && p.shape[p.nd - 1] >= 32) p.form = AFORM_COLUMN;
    else p.form = AFORM_GENERAL;
    const long long per_cta = p.form == AFORM_ROW ? kAWarps : kAThreads;
    const long long base = arg_cdiv(p.n_out, per_cta);
    long long S = 1;
    if (base < kArgTargetCtas && p.L >= 2 * kArgMinChunk)
      S = std::min(std::min(arg_cdiv(kArgTargetCtas, std::max(base, 1ll)), p.L / kArgMinChunk), kArgMaxSplit);
    p.C = S > 1 ? arg_cdiv(arg_cdiv(p.L, S), kArgChunkAlign) * kArgChunkAlign : std::max(p.L, 1ll);
    p.S = (int)std::max(arg_cdiv(p.L, p.C), 1ll);
    p.ctas = p.form == AFORM_ROW ? arg_cdiv(p.n_out * p.S, kAWarps) : base * p.S;
  }
  p.scratch_bytes = p.S > 1 ? (long long)p.S * p.n_out * 16 : 0;
}

void bind_arg_coords(const rb200_index_view& v, int axis, const long long* origin, const long long* gstride, ArgPlan* P) {
  ArgPlan& p = *P;
  if (axis != RB200_ARG_ALL_AXES) {
    p.g0 = origin[axis];
    return;
  }
  p.g0 = 0;
  for (int d = 0; d < v.ndim; ++d) p.g0 += origin[d] * gstride[d];
  // merge neighbours that are contiguous both in memory and in the global flat index
  int nd = 0;
  for (int d = 0; d < v.ndim; ++d) {
    if (v.shape[d] == 1) continue;
    if (nd > 0 && p.stride[nd - 1] == v.stride[d] * v.shape[d] && p.gstride[nd - 1] == gstride[d] * v.shape[d]) {
      p.shape[nd - 1] *= v.shape[d];
      p.stride[nd - 1] = v.stride[d];
      p.gstride[nd - 1] = gstride[d];
      continue;
    }
    p.shape[nd] = v.shape[d];
    p.stride[nd] = v.stride[d];
    p.gstride[nd] = gstride[d];
    ++nd;
  }
  if (nd > 0) p.nd = nd;
}

template <class TS, int OP>
static cudaError_t launch_arg_t(const ArgPlan& P, long long* out_idx, long long* out_key, void* scratch, cudaStream_t s) {
  longlong2* part = (longlong2*)scratch;
  if (P.form == AFORM_GLOBAL) arg_global_kernel<TS, OP><<<(unsigned)P.ctas, kAThreads, 0, s>>>(P, out_idx, out_key, part);
  else if (P.form == AFORM_ROW) arg_row_kernel<TS, OP><<<(unsigned)P.ctas, kAThreads, 0, s>>>(P, out_idx, out_key, part);
  else arg_kept_kernel<TS, OP><<<(unsigned)P.ctas, kAThreads, 0, s>>>(P, out_idx, out_key, part);
  if (P.S > 1) arg_fold_kernel<<<(unsigned)arg_cdiv(P.n_out, kAWarps), kAThreads, 0, s>>>(part, out_idx, out_key, P.n_out, P.S);
  return cudaGetLastError();
}

template <class TS>
static cudaError_t launch_arg_op(const ArgPlan& P, int op, long long* out_idx, long long* out_key, void* scratch, cudaStream_t s) {
  switch (op) {
    case RB200_ARG_MAX: return launch_arg_t<TS, RB200_ARG_MAX>(P, out_idx, out_key, scratch, s);
    case RB200_ARG_MIN: return launch_arg_t<TS, RB200_ARG_MIN>(P, out_idx, out_key, scratch, s);
    case RB200_ARG_NANMAX: return launch_arg_t<TS, RB200_ARG_NANMAX>(P, out_idx, out_key, scratch, s);
    default: return launch_arg_t<TS, RB200_ARG_NANMIN>(P, out_idx, out_key, scratch, s);
  }
}

cudaError_t launch_arg(const ArgPlan& P, int src_dtype, int op, long long* out_idx, long long* out_key, void* scratch, cudaStream_t s) {
  if (P.n_out == 0) return cudaSuccess;
  switch (src_dtype) {
    case RB200_F64: return launch_arg_op<double>(P, op, out_idx, out_key, scratch, s);
    case RB200_F32: return launch_arg_op<float>(P, op, out_idx, out_key, scratch, s);
    case RB200_I64: return launch_arg_op<long long>(P, op, out_idx, out_key, scratch, s);
    default: return launch_arg_op<int>(P, op, out_idx, out_key, scratch, s);
  }
}

}  // namespace rb200
