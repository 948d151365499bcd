// rb200_compact.cu — stream compaction on sm_90a: the positions, values or coordinates of the nonzero elements of a
// strided view, in C order, at positions that depend only on the data.
//
// Layout (include/ramba_b200.h): the view's C-order positions form n_runs runs of run_len positions, and each run is cut
// into chunks of at most kCChunk positions; a chunk never crosses a run.  Chunk (r, c) is q = c * n_runs + r, so that a
// scan along the runs is a column scan of a [cpr][n_runs] block and the last row holds every run's total.
//   * A CTA covers one contiguous range of positions: one chunk when run_len >= kCChunk, otherwise
//     runs_per_cta = kCChunk / run_len whole runs (one chunk each, so short runs cost one CTA per kCChunk positions).
//     (A grid of 8 CTAs per SM walking these ranges measured slower on an H100 80GB HBM3 at 700 W: 0.63 ms against
//     0.51 ms to count 1e9 bool.)
//   * Inside the range every thread reads 16 bytes per pass (EB passes of 16 / EB elements: one 16-byte load when the
//     view is one aligned unit-stride run), keeps one predicate bit per element, and the CTA's exclusive prefix of those
//     bits comes from one packed warp scan (16-bit fields, one per pass) and the warp totals.  Order: pass, thread, lane.
//   * rb200_compact_count writes each chunk's count (the prefix at the next chunk's start minus the prefix at its own).
//   * rb200_compact reads the condition again and sends each selected element to
//     run_base[r] + incl[q] - counts[q] + (its prefix - the prefix at its chunk's start); the positions are first put
//     in rank order in shared memory so that a warp writes 32 consecutive outputs.
// No atomics on data: the position of every element is a function of the condition alone.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>

#include "rb200_compact.h"

namespace rb200 {

constexpr int kCThreads = 256;
constexpr int kCPer = 16;                     // positions per thread
constexpr int kCChunk = kCThreads * kCPer;    // == RB200_COMPACT_CHUNK
static_assert(kCChunk == RB200_COMPACT_CHUNK, "chunk size is part of the ABI");
constexpr int kCWarps = kCThreads / 32;

template <int EB> struct CWord;
template <> struct CWord<1> { using T = unsigned char; };
template <> struct CWord<2> { using T = unsigned short; };
template <> struct CWord<4> { using T = unsigned int; };
template <> struct CWord<8> { using T = unsigned long long; };

// x != 0 on the stored bits: floats drop the sign bit first (-0.0 is zero, NaN is not)
template <int EB, bool FL> __device__ __forceinline__ bool c_nonzero(typename CWord<EB>::T w) {
  if constexpr (FL) return (typename CWord<EB>::T)(w << 1) != 0;
  else return w != 0;
}

// the range of positions [p0, p1) of this CTA, its first run and chunk column, and how many chunks it holds
struct CRange {
  long long p0, p1, r0, c;
  int nq;
};

__device__ __forceinline__ CRange c_range(const CompactPlan& P, long long g) {
  CRange R;
  if (P.run_len >= kCChunk) {
    R.r0 = g / P.cpr;
    R.c = g - R.r0 * P.cpr;
    R.p0 = R.r0 * P.run_len + R.c * kCChunk;
    R.p1 = min(R.p0 + (long long)kCChunk, (R.r0 + 1) * P.run_len);
    R.nq = 1;
  } else {
    R.r0 = g * P.runs_per_cta;
    const long long r1 = min(R.r0 + P.runs_per_cta, P.n_runs);
    R.p0 = R.r0 * P.run_len;
    R.p1 = r1 * P.run_len;
    R.c = 0;
    R.nq = (int)(r1 - R.r0);
  }
  return R;
}

// Shared state of one CTA: per pass and thread the exclusive prefix, per thread the predicate bits.
template <int EB> struct CShared {
  static constexpr int NP = EB;  // passes
  int ex[NP][kCThreads];
  unsigned short mask[kCThreads];
  unsigned long long wt[kCWarps][(NP + 3) / 4];
};

// Phase 1: predicate bits of this thread (bit k * E + u: pass k, lane u) and the exclusive prefix of each pass in *ex;
// the CTA's total in the return value.  Writes S.ex / S.mask and ends with a barrier.
template <int EB, bool FL>
__device__ __forceinline__ int c_scan(const CompactView& V, const CRange& R, CShared<EB>& S, unsigned& bits, int (&ex)[EB]) {
  using W = typename CWord<EB>::T;
  constexpr int E = 16 / EB, NP = EB, NW = (NP + 3) / 4;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const bool vec = V.nd == 1 && V.stride[0] == 1 && (((unsigned long long)(V.base + R.p0 * EB)) & 15) == 0;
  bits = 0;
  unsigned long long pk[NW];
#pragma unroll
  for (int w = 0; w < NW; ++w) pk[w] = 0;
#pragma unroll
  for (int k = 0; k < NP; ++k) {
    const long long p = R.p0 + (long long)k * kCThreads * E + (long long)t * E;
    unsigned m = 0;
    if (vec && p + E <= R.p1) {
      const uint4 v = __ldcs(reinterpret_cast<const uint4*>(V.base + p * EB));
      W w[E];
      memcpy(w, &v, 16);
#pragma unroll
      for (int u = 0; u < E; ++u) m |= (unsigned)c_nonzero<EB, FL>(w[u]) << u;
    } else {
#pragma unroll
      for (int u = 0; u < E; ++u)
        if (p + u < R.p1) m |= (unsigned)c_nonzero<EB, FL>(__ldcs(reinterpret_cast<const W*>(V.base) + c_offset(V, p + u))) << u;
    }
    bits |= m << (k * E);
    pk[k / 4] |= (unsigned long long)__popc(m) << (16 * (k % 4));
  }
  unsigned long long inc[NW];
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    inc[w] = pk[w];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long o = __shfl_up_sync(0xffffffffu, inc[w], d);
      if (lane >= d) inc[w] += o;
    }
    if (lane == 31) S.wt[warp][w] = inc[w];
  }
  __syncthreads();
  int total = 0;
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    unsigned long long before = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < kCWarps; ++i) {
      const unsigned long long x = S.wt[i][w];
      if (i < warp) before += x;
      tot += x;
    }
    const unsigned long long mine = before + inc[w] - pk[w];
#pragma unroll
    for (int f = 0; f < 4; ++f) {
      const int k = w * 4 + f;
      if (k < NP) {
        ex[k] = total + (int)((mine >> (16 * f)) & 0xffff);
        S.ex[k][t] = ex[k];
        total += (int)((tot >> (16 * f)) & 0xffff);
      }
    }
  }
  S.mask[t] = (unsigned short)bits;
  __syncthreads();
  return total;
}

// the CTA prefix at position p0 + rel (rel < kCChunk), from the shared state
template <int EB> __device__ __forceinline__ int c_prefix_at(const CShared<EB>& S, int rel) {
  constexpr int E = 16 / EB;
  const int k = rel / (kCThreads * E), r = rel - k * kCThreads * E, t = r / E, u = r - t * E;
  return S.ex[k][t] + __popc(((unsigned)S.mask[t] >> (k * E)) & ((1u << u) - 1u));
}

template <int EB, bool FL>
__global__ void __launch_bounds__(kCThreads) compact_count_kernel(const __grid_constant__ CompactPlan P, long long* __restrict__ counts) {
  __shared__ CShared<EB> S;
  const CRange R = c_range(P, blockIdx.x);
  unsigned bits;
  int ex[EB];
  const int total = c_scan<EB, FL>(P.cond, R, S, bits, ex);
  if (R.nq == 1) {
    if (threadIdx.x == 0) counts[R.c * P.n_runs + R.r0] = total;
    return;
  }
  const int rl = (int)P.run_len;
  for (int j = threadIdx.x; j < R.nq; j += kCThreads) {
    const int lo = c_prefix_at<EB>(S, j * rl);
    const int hi = j + 1 < R.nq ? c_prefix_at<EB>(S, (j + 1) * rl) : total;
    counts[R.r0 + j] = hi - lo;
  }
}

template <int VEB> __device__ __forceinline__ void c_put_value(const CompactOut& O, long long p, long long dest) {
  using W = typename CWord<VEB>::T;
  reinterpret_cast<W*>(O.out[0])[dest] = __ldcs(reinterpret_cast<const W*>(O.values.base) + c_offset(O.values, p));
}

// MODE: 1, 2, 4, 8 = VALUES of that many bytes; 0 = FLAT; -1 = COORDS
template <int MODE> __device__ __forceinline__ void c_put(const CompactOut& O, long long p, long long dest) {
  if constexpr (MODE > 0) {
    c_put_value<MODE>(O, p, dest);
  } else if constexpr (MODE == 0) {
    long long f = O.g0;
    if (O.k == 1) {
      f += p * O.gstride[0];
    } else {
#pragma unroll
      for (int d = RB200_MAX_DIMS - 1; d > 0; --d) {
        if (d < O.k) {
          const long long q = p / O.cshape[d];
          f += (p - q * O.cshape[d]) * O.gstride[d];
          p = q;
        }
      }
      f += p * O.gstride[0];
    }
    reinterpret_cast<long long*>(O.out[0])[dest] = f;
  } else {
#pragma unroll
    for (int d = RB200_MAX_DIMS - 1; d > 0; --d) {
      if (d < O.k) {
        const long long q = p / O.cshape[d];
        reinterpret_cast<long long*>(O.out[d])[dest] = O.origin[d] + (p - q * O.cshape[d]);
        p = q;
      }
    }
    reinterpret_cast<long long*>(O.out[0])[dest] = O.origin[0] + p;
  }
}

// Phase 2: the selected positions go to shared memory in rank order, so that consecutive threads then write
// consecutive output positions (and read nearly consecutive values).
template <int EB, bool FL, int MODE>
__global__ void __launch_bounds__(kCThreads) compact_kernel(const __grid_constant__ CompactPlan P, const __grid_constant__ CompactOut O,
                                                            const long long* __restrict__ counts, const long long* __restrict__ incl,
                                                            const long long* __restrict__ run_base) {
  __shared__ CShared<EB> S;
  __shared__ unsigned short s_pos[kCChunk];
  constexpr int E = 16 / EB;
  const CRange R = c_range(P, blockIdx.x);
  unsigned bits;
  int ex[EB];
  const int total = c_scan<EB, FL>(P.cond, R, S, bits, ex);
#pragma unroll
  for (int k = 0; k < EB; ++k) {
    const unsigned mk = (bits >> (k * E)) & ((1u << E) - 1u);
    const int rel0 = k * kCThreads * E + (int)threadIdx.x * E;
    for (unsigned m = mk; m; m &= m - 1) {
      const int u = __ffs(m) - 1;
      s_pos[ex[k] + __popc(mk & ((1u << u) - 1u))] = (unsigned short)(rel0 + u);
    }
  }
  long long off = 0;  // one chunk: the output position of its first selected element
  if (R.nq == 1) {
    const long long q = R.c * P.n_runs + R.r0;
    off = run_base[R.r0] + incl[q] - counts[q];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < total; i += kCThreads) {
    const int rel = s_pos[i];
    long long dest = off + i;
    if (R.nq > 1) {  // short runs: chunk j = rel / run_len is run r0 + j
      const int j = rel / (int)P.run_len;
      const long long r = R.r0 + j;
      dest += run_base[r] + incl[r] - counts[r] - c_prefix_at<EB>(S, j * (int)P.run_len);
    }
    c_put<MODE>(O, R.p0 + rel, dest);
  }
}

// ---- host: plan and dispatch --------------------------------------------------------------------------------------------
static long long c_cdiv(long long a, long long b) { return (a + b - 1) / b; }

CompactView make_compact_view(const rb200_index_view& v) {
  CompactView c;
  c.base = (const char*)v.base;
  c.eb = v.elem_bytes;
  c.nd = 0;
  for (int d = 0; d < v.ndim; ++d) {
    if (v.shape[d] == 1) continue;
    if (c.nd > 0 && c.stride[c.nd - 1] == v.stride[d] * v.shape[d]) {
      c.shape[c.nd - 1] *= v.shape[d];
      c.stride[c.nd - 1] = v.stride[d];
      continue;
    }
    c.shape[c.nd] = v.shape[d];
    c.stride[c.nd] = v.stride[d];
    ++c.nd;
  }
  if (c.nd == 0) {
    c.shape[0] = 1;
    c.stride[0] = 1;
    c.nd = 1;
  }
  return c;
}

void make_compact_plan(const rb200_index_view& cond, long long run_len, CompactPlan* P) {
  CompactPlan& p = *P;
  p.cond = make_compact_view(cond);
  p.n = 1;
  for (int d = 0; d < cond.ndim; ++d) p.n *= cond.shape[d];
  p.run_len = run_len;
  p.n_runs = run_len > 0 ? p.n / run_len : 0;
  p.cpr = c_cdiv(run_len, kCChunk);
  p.runs_per_cta = run_len >= kCChunk ? 1 : kCChunk / std::max(run_len, 1ll);
  p.ctas = run_len >= kCChunk ? p.n_runs * p.cpr : c_cdiv(p.n_runs, p.runs_per_cta);
}

template <int EB, bool FL> static cudaError_t count_t(const CompactPlan& P, long long* counts, cudaStream_t s) {
  compact_count_kernel<EB, FL><<<(unsigned)P.ctas, kCThreads, 0, s>>>(P, counts);
  return cudaGetLastError();
}

cudaError_t launch_compact_count(const CompactPlan& P, bool is_float, long long* counts, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  switch (P.cond.eb) {
    case 1: return count_t<1, false>(P, counts, s);
    case 2: return count_t<2, false>(P, counts, s);
    case 4: return is_float ? count_t<4, true>(P, counts, s) : count_t<4, false>(P, counts, s);
    default: return is_float ? count_t<8, true>(P, counts, s) : count_t<8, false>(P, counts, s);
  }
}

template <int EB, bool FL, int MODE>
static cudaError_t compact_t(const CompactPlan& P, const CompactOut& O, const long long* counts, const long long* incl, const long long* run_base,
                             cudaStream_t s) {
  compact_kernel<EB, FL, MODE><<<(unsigned)P.ctas, kCThreads, 0, s>>>(P, O, counts, incl, run_base);
  return cudaGetLastError();
}

template <int EB, bool FL>
static cudaError_t compact_mode(const CompactPlan& P, const CompactOut& O, const long long* counts, const long long* incl, const long long* run_base,
                                cudaStream_t s) {
  if (O.form == RB200_COMPACT_FLAT) return compact_t<EB, FL, 0>(P, O, counts, incl, run_base, s);
  if (O.form == RB200_COMPACT_COORDS) return compact_t<EB, FL, -1>(P, O, counts, incl, run_base, s);
  switch (O.values.eb) {
    case 1: return compact_t<EB, FL, 1>(P, O, counts, incl, run_base, s);
    case 2: return compact_t<EB, FL, 2>(P, O, counts, incl, run_base, s);
    case 4: return compact_t<EB, FL, 4>(P, O, counts, incl, run_base, s);
    default: return compact_t<EB, FL, 8>(P, O, counts, incl, run_base, s);
  }
}

cudaError_t launch_compact(const CompactPlan& P, bool is_float, const long long* counts, const long long* incl, const long long* run_base,
                           const CompactOut& O, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  switch (P.cond.eb) {
    case 1: return compact_mode<1, false>(P, O, counts, incl, run_base, s);
    case 2: return compact_mode<2, false>(P, O, counts, incl, run_base, s);
    case 4: return is_float ? compact_mode<4, true>(P, O, counts, incl, run_base, s) : compact_mode<4, false>(P, O, counts, incl, run_base, s);
    default: return is_float ? compact_mode<8, true>(P, O, counts, incl, run_base, s) : compact_mode<8, false>(P, O, counts, incl, run_base, s);
  }
}

}  // namespace rb200
