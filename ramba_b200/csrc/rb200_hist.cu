// rb200_hist.cu — binning on sm_90a: histograms of a strided view (uniform bins restating NumPy's fast path, explicit
// edges, integer bins) with privatised shared-memory bins, and the binary search of every element in a sorted table.
//
// Histogram (include/ramba_b200.h states the contract and the fold order):
//   * CTA c owns the C-order positions [c * chunk, (c + 1) * chunk); chunk is a whole number of kHUnit positions chosen
//     from n alone, so at most kHMaxCtas CTAs run.  A step of the CTA covers kHThreads * E * kHU positions (E = 16 / element
//     bytes): warp w takes its 32 * E * kHU of them, in kHU groups of 32 lanes * E consecutive positions, each group one
//     16-byte load per lane when the view is one aligned unit-stride run.
//   * Counts, shared form: one row of 32-bit counters in shared memory per CTA.  For every (group, element) a warp whose
//     32 lanes fall into one bin adds 32 with one shared atomic (data skewed into one bin), otherwise each lane adds its
//     own element.  At the end every nonzero counter is added to the output with one int64 atomic (integers: the order
//     does not matter).
//   * Counts, global form (the row does not fit): the same, with int64 atomics straight into the output.
//   * Weights, shared form: one float64 row per warp.  The lanes that fall into one bin find each other with
//     __match_any_sync, and the lowest of them adds the group's weights in
//     ascending lane order and then adds that to its warp's row (plain load / add / store: the row is the warp's own).
//     The CTA's rows are summed in warp order from +0.0 into scratch[c][b]; a second launch folds scratch in CTA order
//     from +0.0.  No float atomics: the sums depend on the data, n, B and the element size only.
//   * Weights, slab form: the bins are cut into slabs that fit; one pass of the shared form per slab.
// Bin search: a thread per element, the table staged in shared memory when it fits, read through the read-only path
// otherwise; NumPy's order (NaN after every number).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <type_traits>

#include "rb200_hist.h"

namespace rb200 {

constexpr int kHThreads = 256;
constexpr int kHWarps = kHThreads / 32;
constexpr int kHU = 4;                   // 16-byte groups per lane per step
constexpr long long kHUnit = 8192;       // chunk granule: whole CTA steps for 4- and 8-byte elements
constexpr long long kHMaxCtas = 1056;
constexpr long long kHShared = 96 * 1024;  // dynamic shared memory budget of one CTA
constexpr int kSThreads = 256;
static_assert(kHUnit % (kHThreads * 4 * kHU) == 0 && kHUnit % (kHThreads * 2 * kHU) == 0, "a chunk is whole CTA steps");

// ---- device helpers ------------------------------------------------------------------------------------------------------
template <class T> __device__ __forceinline__ double h_f64(T x) {
  if constexpr (std::is_same<T, long long>::value) return __ll2double_rn(x);
  else return (double)x;
}
template <class T> __device__ __forceinline__ float h_f32(T x) {
  if constexpr (std::is_same<T, double>::value) return __double2float_rn(x);
  else if constexpr (std::is_same<T, long long>::value) return __ll2float_rn(x);
  else if constexpr (std::is_same<T, int>::value) return __int2float_rn(x);
  else return x;
}
template <class C, class T> __device__ __forceinline__ C h_to(T x) {
  if constexpr (std::is_same<C, double>::value) return h_f64(x);
  else if constexpr (std::is_same<C, float>::value) return h_f32(x);
  else return (long long)x;
}

// NumPy's sort order: a < b, with NaN after every number
template <class C> __device__ __forceinline__ bool h_lt(C a, C b) {
  if constexpr (std::is_floating_point<C>::value) return a < b || (b != b && a == a);
  else return a < b;
}

template <class C> __device__ __forceinline__ C h_tab(const C* t, long long i, bool shared) { return shared ? t[i] : __ldg(t + i); }

// left: the number of t[i] with lt(t[i], x); right: the number with !lt(x, t[i]) (t sorted in that order)
template <class C> __device__ __forceinline__ long long h_search(const C* t, long long n, C x, bool right, bool shared) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    const C v = h_tab(t, mid, shared);
    if (right ? !h_lt(x, v) : h_lt(v, x)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// first <= x (ge) or x <= last in dtype dt (F64, F32 or I64)
template <class T> __device__ __forceinline__ bool h_bound(T x, int dt, double b, long long bi, bool ge) {
  if (dt == RB200_I64) {
    if constexpr (std::is_integral<T>::value) return ge ? (long long)x >= bi : (long long)x <= bi;
    else return false;
  }
  if (dt == RB200_F32) {
    const float v = h_f32(x), c = (float)b;
    return ge ? v >= c : v <= c;
  }
  const double v = h_f64(x);
  return ge ? v >= b : v <= b;
}

// NumPy's fix-ups of the estimated index against the edge table; -2: an index outside [0, B)
template <class E> __device__ __forceinline__ long long h_fixup(E xe, long long idx, const E* e, long long B, bool shared) {
  if (idx == B) --idx;
  if (idx < 0 || idx >= B) return -2;
  if (xe < h_tab(e, idx, shared)) --idx;
  if (idx != B - 1 && xe >= h_tab(e, idx + 1, shared)) ++idx;
  return idx < 0 ? -2 : idx;
}

// numpy/lib/_histograms_impl.py::histogram, the equal-bins path, on one element: -1 not kept, -2 bad, else the bin
template <class T> __device__ __forceinline__ long long h_uniform(T x, const rb200_bin_table& Tb, const void* tab, bool shared) {
  if (!h_bound(x, Tb.lo_dtype, Tb.lo, Tb.lo_i, true) || !h_bound(x, Tb.hi_dtype, Tb.hi, Tb.hi_i, false)) return -1;
  const long long B = Tb.n_bins;
  if (Tb.edge_dtype == RB200_F64) {  // (the subtraction and the division are then float64 too)
    const double xe = h_f64(x);
    const long long idx = __double2ll_rz(__dmul_rn(__ddiv_rn(__dsub_rn(xe, Tb.first), Tb.denom), (double)B));
    return h_fixup(xe, idx, (const double*)tab, B, shared);
  }
  const float xe = h_f32(x);
  long long idx;
  if (Tb.sub_dtype == RB200_F32) {
    const float s = __fsub_rn(xe, (float)Tb.first);
    if (Tb.div_dtype == RB200_F32) idx = __float2ll_rz(__fmul_rn(__fdiv_rn(s, (float)Tb.denom), (float)B));
    else idx = __double2ll_rz(__dmul_rn(__ddiv_rn((double)s, Tb.denom), (double)B));
  } else {
    idx = __double2ll_rz(__dmul_rn(__ddiv_rn(__dsub_rn((double)xe, Tb.first), Tb.denom), (double)B));
  }
  return h_fixup(xe, idx, (const float*)tab, B, shared);
}

// explicit edges: e[i] <= x < e[i+1], the last bin closed, in NumPy's order; -1 outside
template <class C, class T> __device__ __forceinline__ long long h_edges(T x, const C* e, long long B, bool shared) {
  const C c = h_to<C>(x);
  const long long j = h_search(e, B, c, true, shared);
  if (j == 0) return -1;
  if (j < B) return j - 1;
  return h_lt(h_tab(e, B, shared), c) ? -1 : B - 1;
}

template <class T> __device__ __forceinline__ long long h_bin(T x, const rb200_bin_table& Tb, const void* tab, bool shared) {
  if (Tb.form == RB200_BINS_UNIFORM) return h_uniform(x, Tb, tab, shared);
  if (Tb.form == RB200_BINS_EDGES) {
    if (Tb.edge_dtype == RB200_F64) return h_edges<double>(x, (const double*)tab, Tb.n_bins, shared);
    if (Tb.edge_dtype == RB200_F32) return h_edges<float>(x, (const float*)tab, Tb.n_bins, shared);
    return h_edges<long long>(x, (const long long*)tab, Tb.n_bins, shared);
  }
  if constexpr (std::is_integral<T>::value) {
    const long long v = (long long)x;
    return v < 0 || v >= Tb.n_bins ? -2 : v;
  } else {
    return -2;
  }
}

__device__ __forceinline__ double h_weight(const CompactView& w, int dt, long long p) {
  const long long o = c_offset(w, p);
  switch (dt) {
    case RB200_F64: return __ldcs(reinterpret_cast<const double*>(w.base) + o);
    case RB200_F32: return (double)__ldcs(reinterpret_cast<const float*>(w.base) + o);
    case RB200_I64: return __ll2double_rn(__ldcs(reinterpret_cast<const long long*>(w.base) + o));
    default: return (double)__ldcs(reinterpret_cast<const int*>(w.base) + o);
  }
}

struct HistArgs {
  HistPlan P;
  rb200_bin_table T;
  long long lo, nb;  // this pass: bins [lo, lo + nb)
  void* out;
  unsigned long long* bad;
  double* scratch;
};

// the byte offset of the staged edge table in shared memory (after the rows and the weight staging)
__host__ __device__ inline long long hist_table_offset(bool weighted, int form, long long slab) {
  const long long rows = weighted ? (kHWarps * slab + kHWarps * 32) * 8 : (form == HIST_GLOBAL ? 0 : slab * 4);
  return (rows + 15) / 16 * 16;
}

template <class T, bool W, bool GLOBAL>
__global__ void __launch_bounds__(kHThreads, 2) hist_kernel(const __grid_constant__ HistArgs A) {
  extern __shared__ __align__(16) unsigned char h_smem[];
  constexpr int E = 16 / sizeof(T);
  const HistPlan& P = A.P;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const long long S = P.slab, nb = A.nb, lo = A.lo;
  double* rows_d = reinterpret_cast<double*>(h_smem);
  double* s_w = rows_d + kHWarps * S + warp * 32;
  unsigned* rows_u = reinterpret_cast<unsigned*>(h_smem);
  const void* tab = A.T.edges;
  if (P.table_shared) {
    unsigned* d = reinterpret_cast<unsigned*>(h_smem + hist_table_offset(W, P.form, S));
    const unsigned* s = reinterpret_cast<const unsigned*>(A.T.edges);
    for (long long i = t; i < P.table_bytes / 4; i += kHThreads) d[i] = __ldg(s + i);
    tab = d;
  }
  if constexpr (W) {
    for (long long i = t; i < kHWarps * S; i += kHThreads) rows_d[i] = 0.0;
  } else if constexpr (!GLOBAL) {
    for (long long i = t; i < S; i += kHThreads) rows_u[i] = 0u;
  }
  __syncthreads();
  const bool sh = P.table_shared;
  const long long p0 = (long long)blockIdx.x * P.chunk, p1 = min(p0 + P.chunk, P.n);
  unsigned long long bad = 0;
  for (long long b0 = p0 + (long long)warp * 32 * E * kHU; b0 < p1; b0 += (long long)kHThreads * E * kHU) {
    T x[kHU][E];
#pragma unroll
    for (int k = 0; k < kHU; ++k) {
      const long long base = b0 + (long long)(k * 32 + lane) * E;
      if (P.vec && base + E <= p1) {
        const uint4 v = __ldcs(reinterpret_cast<const uint4*>(P.src.base + base * (long long)sizeof(T)));
        memcpy(x[k], &v, 16);
      } else {
#pragma unroll
        for (int u = 0; u < E; ++u)
          x[k][u] = base + u < p1 ? __ldcs(reinterpret_cast<const T*>(P.src.base) + c_offset(P.src, base + u)) : T(0);
      }
    }
#pragma unroll
    for (int k = 0; k < kHU; ++k) {
#pragma unroll
      for (int u = 0; u < E; ++u) {
        const long long p = b0 + (long long)(k * 32 + lane) * E + u;
        long long bin = p < p1 ? h_bin(x[k][u], A.T, tab, sh) : -1;
        if (bin == -2) {
          bad += lo == 0;
          bin = -1;
        }
        if (bin >= lo + nb) bin = -1;
        const unsigned key = bin >= lo ? (unsigned)(bin - lo) : 0xffffffffu;
        if constexpr (W) {
          const unsigned m = __match_any_sync(0xffffffffu, key);
          const bool leader = key != 0xffffffffu && lane == __ffs(m) - 1;
          s_w[lane] = key != 0xffffffffu ? h_weight(P.w, P.w_dtype, p) : 0.0;
          __syncwarp();
          if (leader) {
            double s = s_w[lane];
            for (unsigned r = m & (m - 1); r; r &= r - 1) s += s_w[__ffs(r) - 1];
            rows_d[warp * S + key] += s;
          }
          __syncwarp();
        } else {
          const unsigned add = warp_bin_share(key, lane);
          if (add) {
            if constexpr (GLOBAL) atomicAdd(reinterpret_cast<unsigned long long*>(A.out) + bin, (unsigned long long)add);
            else atomicAdd(rows_u + key, add);
          }
        }
      }
    }
  }
  for (int d = 16; d > 0; d >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, d);
  if (lane == 0 && bad) atomicAdd(A.bad, bad);
  if constexpr (GLOBAL) return;
  __syncthreads();
  for (long long b = t; b < nb; b += kHThreads) {
    if constexpr (W) {
      double v = 0.0;
#pragma unroll
      for (int w = 0; w < kHWarps; ++w) v += rows_d[w * S + b];
      A.scratch[(long long)blockIdx.x * nb + b] = v;
    } else {
      const unsigned c = rows_u[b];
      if (c) atomicAdd(reinterpret_cast<unsigned long long*>(A.out) + lo + b, (unsigned long long)c);
    }
  }
}

// out[lo + b] = +0.0 + scratch[0][b] + scratch[1][b] + ... in CTA order
__global__ void __launch_bounds__(kHThreads) hist_fold_kernel(const double* __restrict__ scratch, long long ctas, long long nb, double* __restrict__ out) {
  const long long b = (long long)blockIdx.x * kHThreads + threadIdx.x;
  if (b >= nb) return;
  double v = 0.0;
  long long c = 0;
  for (; c + 8 <= ctas; c += 8) {
    double r[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) r[i] = scratch[(c + i) * nb + b];
#pragma unroll
    for (int i = 0; i < 8; ++i) v += r[i];
  }
  for (; c < ctas; ++c) v += scratch[c * nb + b];
  out[b] = v;
}

struct SearchArgs {
  SearchPlan P;
  const void* table;
  long long* out;
};

template <class T, class C>
__global__ void __launch_bounds__(kSThreads) search_kernel(const __grid_constant__ SearchArgs A) {
  extern __shared__ __align__(16) unsigned char h_smem[];
  const C* tab = reinterpret_cast<const C*>(A.table);
  if (A.P.table_shared) {
    C* d = reinterpret_cast<C*>(h_smem);
    for (long long i = threadIdx.x; i < A.P.n_tab; i += kSThreads) d[i] = __ldg(tab + i);
    tab = d;
    __syncthreads();
  }
  const bool sh = A.P.table_shared, right = A.P.side == RB200_SEARCH_RIGHT;
  for (long long p = (long long)blockIdx.x * kSThreads + threadIdx.x; p < A.P.n; p += (long long)gridDim.x * kSThreads) {
    const T x = __ldcs(reinterpret_cast<const T*>(A.P.src.base) + c_offset(A.P.src, p));
    A.out[p] = h_search(tab, A.P.n_tab, h_to<C>(x), right, sh);
  }
}

// ---- host: plans and dispatch --------------------------------------------------------------------------------------------
static long long h_cdiv(long long a, long long b) { return (a + b - 1) / b; }
static int h_esz(int dt) { return dt == RB200_F32 ? 4 : 8; }

const char* hist_form_name(int form) { return form == HIST_SHARED ? "shared" : form == HIST_GLOBAL ? "global" : "slab"; }

void make_hist_plan(const rb200_index_view& src, bool weighted, const rb200_bin_table& T, HistPlan* P) {
  HistPlan& p = *P;
  p.src = make_compact_view(src);
  p.weighted = weighted;
  p.n = 1;
  for (int d = 0; d < src.ndim; ++d) p.n *= src.shape[d];
  p.B = T.n_bins;
  p.ctas = p.n ? std::min(h_cdiv(p.n, kHUnit), kHMaxCtas) : 0;
  p.chunk = p.n ? h_cdiv(h_cdiv(p.n, p.ctas), kHUnit) * kHUnit : 0;
  p.ctas = p.n ? h_cdiv(p.n, p.chunk) : 0;
  p.vec = p.src.nd == 1 && p.src.stride[0] == 1 && (((unsigned long long)p.src.base) & 15) == 0;
  p.table_bytes = T.form == RB200_BINS_INTEGER ? 0 : (p.B + 1) * h_esz(T.edge_dtype);
  if (!weighted) {
    p.form = p.B * 4 <= kHShared ? HIST_SHARED : HIST_GLOBAL;
    p.slab = p.form == HIST_SHARED ? p.B : 0;
  } else {
    const long long fit = (kHShared - kHWarps * 32 * 8) / (kHWarps * 8);
    p.form = p.B <= fit ? HIST_SHARED : HIST_SLAB;
    p.slab = std::min(p.B, fit);
  }
  p.passes = weighted ? h_cdiv(p.B, p.slab) : 1;
  const long long toff = hist_table_offset(weighted, p.form, p.slab);
  p.table_shared = p.table_bytes > 0 && toff + p.table_bytes <= kHShared;
  p.shared_bytes = p.form == HIST_GLOBAL && !p.table_shared ? 0 : toff + (p.table_shared ? p.table_bytes : 0);
  p.scratch_bytes = weighted ? p.ctas * p.slab * 8 : 0;
}

void make_search_plan(const rb200_index_view& src, long long n_tab, int tab_dtype, SearchPlan* P) {
  SearchPlan& p = *P;
  p.src = make_compact_view(src);
  p.n = 1;
  for (int d = 0; d < src.ndim; ++d) p.n *= src.shape[d];
  p.n_tab = n_tab;
  p.tab_dtype = tab_dtype;
  p.ctas = p.n ? std::min(h_cdiv(p.n, kSThreads * 4), kHMaxCtas) : 0;
  const long long tb = n_tab * h_esz(tab_dtype);
  p.table_shared = tb > 0 && tb <= kHShared;
  p.shared_bytes = p.table_shared ? tb : 0;
}

template <class T, bool W, bool GLOBAL> static cudaError_t hist_t(const HistArgs& A, cudaStream_t s) {
  const auto k = hist_kernel<T, W, GLOBAL>;
  if (const cudaError_t e = allow_shared(k, A.P.shared_bytes)) return e;
  k<<<(unsigned)A.P.ctas, kHThreads, (size_t)A.P.shared_bytes, s>>>(A);
  return cudaGetLastError();
}

template <class T> static cudaError_t hist_dtype(const HistArgs& A, cudaStream_t s) {
  if (A.P.weighted) return hist_t<T, true, false>(A, s);
  if (A.P.form == HIST_GLOBAL) return hist_t<T, false, true>(A, s);
  return hist_t<T, false, false>(A, s);
}

cudaError_t launch_histogram(const HistPlan& P, const rb200_bin_table& T, const rb200_index_view* weights, void* out, unsigned long long* bad,
                             void* scratch, cudaStream_t s) {
  const size_t out_bytes = (size_t)P.B * 8;
  if (P.n == 0 || !P.weighted) {
    const cudaError_t e = cudaMemsetAsync(out, 0, out_bytes, s);  // (all-zero bits: int64 0 and float64 +0.0)
    if (e != cudaSuccess || P.n == 0) return e;
  }
  HistArgs A;
  A.P = P;
  if (weights) A.P.w = make_compact_view(*weights);
  A.T = T;
  A.out = out;
  A.bad = bad;
  A.scratch = reinterpret_cast<double*>(scratch);
  for (long long pass = 0; pass < P.passes; ++pass) {
    A.lo = pass * (P.weighted ? P.slab : 0);
    A.nb = P.weighted ? std::min(P.slab, P.B - A.lo) : P.B;
    cudaError_t e;
    switch (P.src_dtype) {
      case RB200_F64: e = hist_dtype<double>(A, s); break;
      case RB200_F32: e = hist_dtype<float>(A, s); break;
      case RB200_I64: e = hist_dtype<long long>(A, s); break;
      default: e = hist_dtype<int>(A, s); break;
    }
    if (e != cudaSuccess) return e;
    if (P.weighted) {
      hist_fold_kernel<<<(unsigned)h_cdiv(A.nb, kHThreads), kHThreads, 0, s>>>(A.scratch, P.ctas, A.nb, reinterpret_cast<double*>(out) + A.lo);
      if (const cudaError_t e2 = cudaGetLastError()) return e2;
    }
  }
  return cudaSuccess;
}

template <class T, class C> static cudaError_t search_t(const SearchArgs& A, cudaStream_t s) {
  const auto k = search_kernel<T, C>;
  if (const cudaError_t e = allow_shared(k, A.P.shared_bytes)) return e;
  k<<<(unsigned)A.P.ctas, kSThreads, (size_t)A.P.shared_bytes, s>>>(A);
  return cudaGetLastError();
}

template <class T> static cudaError_t search_dtype(const SearchArgs& A, cudaStream_t s) {
  if (A.P.tab_dtype == RB200_F64) return search_t<T, double>(A, s);
  if (A.P.tab_dtype == RB200_F32) return search_t<T, float>(A, s);
  return search_t<T, long long>(A, s);
}

cudaError_t launch_bin_search(const SearchPlan& P, const void* table, long long* out, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  SearchArgs A;
  A.P = P;
  A.table = table;
  A.out = out;
  switch (P.src_dtype) {
    case RB200_F64: return search_dtype<double>(A, s);
    case RB200_F32: return search_dtype<float>(A, s);
    case RB200_I64: return search_dtype<long long>(A, s);
    default: return search_dtype<int>(A, s);
  }
}

}  // namespace rb200
