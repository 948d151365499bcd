// rb200_select.cu — order statistics on sm_90a: the k-th smallest keys of the segments of a strided view, by radix select
// (include/ramba_b200.h states the key map, the two forms and the pass contract).
//
//   * Key map: s_key below, the one device statement of the header's map.
//   * `pass` form, count: CTA c covers segment c / cps, C-order positions [(c % cps) * chunk, ...) of it (chunk a whole
//     number of kQUnit positions chosen from the shapes alone).  A step of the CTA covers kQThreads * E * kQU positions
//     (E = 16 / element bytes): warp w takes 32 * E * kQU of them, kQU groups of 32 lanes * E consecutive positions,
//     one 16-byte load per lane when the view is one aligned unit-stride run.  Each key that matches one of the
//     segment's count rows (its prefix, the bits chosen so far) is counted in a 32-bit shared-memory counter of its row
//     and digit, with hist_kernel's warp aggregation (warp_bin_share); the CTA adds its nonzero counters to the int64
//     counts with one atomic each.  `rows` count rows fit in shared memory per launch; more take `groups` launches.
//   * Candidate compaction: in APPEND mode each warp appends its matching keys with one atomic on the counter and one
//     ballot (order is irrelevant to ranks, so no scan is needed); CAND mode reads those keys as 16-byte vectors.
//   * choose: one warp per segment; for each target a warp-wide scan of its row's buckets, 32 at a time.
//   * `row` form: one CTA per segment loads the segment's keys into shared memory once and selects each target by 8-bit
//     digits there, with the same warp-aggregated counters.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <type_traits>

#include "rb200_hist.h"
#include "rb200_select.h"

namespace rb200 {

constexpr int kQThreads = 256;
constexpr int kQWarps = kQThreads / 32;
constexpr int kQU = 4;                    // 16-byte groups per lane per step
constexpr long long kQUnit = 8192;        // chunk granule: whole CTA steps for 4- and 8-byte elements
constexpr long long kQMaxCtas = 1056;
constexpr long long kQShared = 96 * 1024;  // dynamic shared memory budget of one CTA
constexpr int kQMaxRows = (int)(kQShared / (256 * 4));
constexpr int kQRowHist = 256 * 4;         // row form: one 8-bit digit's counters
constexpr int kQChooseWarps = 4;
constexpr unsigned kNone = 0xffffffffu;
static_assert(kQUnit % (kQThreads * 4 * kQU) == 0 && kQUnit % (kQThreads * 2 * kQU) == 0, "a chunk is whole CTA steps");

// ---- the key map (include/ramba_b200.h) ----------------------------------------------------------------------------------
template <class T> __device__ __forceinline__ unsigned long long s_key(T x) {
  if constexpr (std::is_same<T, double>::value) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(x);
    if (x != x) return ~0ull;
    return (u >> 63) ? ~u : u | (1ull << 63);
  } else if constexpr (std::is_same<T, float>::value) {
    const unsigned u = __float_as_uint(x);
    if (x != x) return 0xffffffffull;
    return (u >> 31) ? (unsigned long long)(~u) : (unsigned long long)(u | 0x80000000u);
  } else if constexpr (std::is_same<T, long long>::value) {
    return (unsigned long long)x ^ (1ull << 63);
  } else {
    return (unsigned long long)((unsigned)x ^ 0x80000000u);
  }
}

template <class T> __host__ __device__ constexpr unsigned long long s_nan_key() { return sizeof(T) == 8 ? ~0ull : 0xffffffffull; }

// the state row of the view's segment s
__device__ __forceinline__ long long s_row(const rb200_select_state& S, long long s) {
  if (S.seg_dims == 0) return s;
  long long g = S.seg_base;
  for (int d = S.seg_dims - 1; d >= 0; --d) {
    const long long q = s / S.seg_shape[d];
    g += (s - q * S.seg_shape[d]) * S.seg_gstride[d];
    s = q;
  }
  return g;
}

template <class T> __device__ __forceinline__ T s_load(const CompactView& v, long long p) {
  return __ldcs(reinterpret_cast<const T*>(v.base) + c_offset(v, p));
}

// ---- pass form ----------------------------------------------------------------------------------------------------------
struct SelCountArgs {
  SelectPlan P;
  rb200_select_state S;
  int pass, shift, width;
  unsigned long long mask;  // the chosen bits (0 in pass 0)
  long long j0;             // this launch's first count row
  long long cchunk;         // CAND: keys per CTA
  bool count_nan;
};

template <class T, int MODE>
__global__ void __launch_bounds__(kQThreads) select_count_kernel(const __grid_constant__ SelCountArgs A) {
  extern __shared__ __align__(16) unsigned q_rows[];
  __shared__ unsigned long long s_pref[kQMaxRows];
  constexpr bool CAND = MODE == RB200_SELECT_CAND;
  constexpr int E = CAND ? 2 : 16 / (int)sizeof(T);
  const SelectPlan& P = A.P;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const long long seg = CAND ? 0 : (long long)blockIdx.x / P.cps, gseg = s_row(A.S, seg);
  const long long K = A.S.targets, nb = 1ll << A.width;
  const long long total = A.pass == 0 ? 1 : A.S.n_slots[gseg];
  const int nr = (int)min(total - A.j0, P.rows);
  if (nr <= 0) return;
  for (int i = t; i < nr; i += kQThreads) s_pref[i] = A.pass == 0 ? 0ull : A.S.slot_key[gseg * K + A.j0 + i];
  for (long long i = t; i < nr * nb; i += kQThreads) q_rows[i] = 0u;
  __syncthreads();
  long long p0, p1;
  if constexpr (CAND) {
    const long long n = min((long long)*A.S.cand_n, (long long)A.S.cand_cap);
    p0 = (long long)blockIdx.x * A.cchunk;
    p1 = min(p0 + A.cchunk, n);
  } else {
    p0 = seg * P.L + ((long long)blockIdx.x % P.cps) * P.chunk;
    p1 = min(p0 + P.chunk, (seg + 1) * P.L);
  }
  long long nans = 0;
  for (long long b0 = p0 + (long long)warp * 32 * E * kQU; b0 < p1; b0 += (long long)kQThreads * E * kQU) {
    unsigned long long key[kQU][E];
#pragma unroll
    for (int k = 0; k < kQU; ++k) {
      const long long base = b0 + (long long)(k * 32 + lane) * E;
      if constexpr (CAND) {
        if (base + E <= p1) {
          const ulonglong2 v = __ldcs(reinterpret_cast<const ulonglong2*>(A.S.cand + base));
          key[k][0] = v.x;
          key[k][1] = v.y;
        } else {
#pragma unroll
          for (int u = 0; u < E; ++u) key[k][u] = base + u < p1 ? __ldcs(A.S.cand + base + u) : 0ull;
        }
      } else if (P.vec && base + E <= p1) {
        const uint4 v = __ldcs(reinterpret_cast<const uint4*>(P.src.base + base * (long long)sizeof(T)));
        T x[E];
        memcpy(x, &v, 16);
#pragma unroll
        for (int u = 0; u < E; ++u) key[k][u] = s_key(x[u]);
      } else {
#pragma unroll
        for (int u = 0; u < E; ++u) key[k][u] = base + u < p1 ? s_key(s_load<T>(P.src, base + u)) : 0ull;
      }
    }
#pragma unroll
    for (int k = 0; k < kQU; ++k) {
#pragma unroll
      for (int u = 0; u < E; ++u) {
        const bool valid = b0 + (long long)(k * 32 + lane) * E + u < p1;
        const unsigned long long kk = key[k][u];
        if (A.count_nan && valid && kk == s_nan_key<T>()) ++nans;
        unsigned bin = kNone;
        if (valid) {
          for (int j = 0; j < nr; ++j) {
            if ((kk & A.mask) == s_pref[j]) {
              bin = (unsigned)(j * nb + (long long)((kk >> A.shift) & (unsigned long long)(nb - 1)));
              break;
            }
          }
        }
        const unsigned add = warp_bin_share(bin, lane);
        if (add) atomicAdd(q_rows + bin, add);
        if constexpr (MODE == RB200_SELECT_APPEND) {
          const unsigned m = __ballot_sync(0xffffffffu, bin != kNone);
          if (m) {
            const int leader = __ffs(m) - 1;
            unsigned long long at = 0;
            if (lane == leader) at = atomicAdd(reinterpret_cast<unsigned long long*>(A.S.cand_n), (unsigned long long)__popc(m));
            at = __shfl_sync(0xffffffffu, at, leader) + __popc(m & ((1u << lane) - 1u));
            if (bin != kNone && (long long)at < A.S.cand_cap) A.S.cand[at] = kk;
          }
        }
      }
    }
  }
  if (A.count_nan) {
    for (int d = 16; d > 0; d >>= 1) nans += __shfl_xor_sync(0xffffffffu, nans, d);
    if (lane == 0 && nans) atomicAdd(reinterpret_cast<unsigned long long*>(A.S.nans + gseg), (unsigned long long)nans);
  }
  __syncthreads();
  for (long long i = t; i < nr * nb; i += kQThreads) {
    const unsigned c = q_rows[i];
    if (c) {
      const long long j = i / nb, b = i - j * nb;
      atomicAdd(reinterpret_cast<unsigned long long*>(A.S.counts + ((gseg * K + A.j0 + j) << P.digit) + b), (unsigned long long)c);
    }
  }
}

struct SelChooseArgs {
  rb200_select_state S;
  int pass, shift, width, digit;
};

// one warp per segment: each target's bucket, residual rank and key bits; then the targets' shared count rows
__global__ void __launch_bounds__(kQChooseWarps * 32) select_choose_kernel(const __grid_constant__ SelChooseArgs A) {
  const int lane = threadIdx.x & 31;
  const long long seg = (long long)blockIdx.x * kQChooseWarps + (threadIdx.x >> 5);
  if (seg >= A.S.segments) return;
  const long long K = A.S.targets, nb = 1ll << A.width;
  int n_new = 0;
  long long matched = 0;
  for (long long k = 0; k < K; ++k) {
    const long long tk = seg * K + k;
    const long long row = A.pass == 0 ? 0 : A.S.slot[tk];
    const long long* h = reinterpret_cast<const long long*>(A.S.counts) + ((seg * K + row) << A.digit);
    long long r = A.S.rank[tk], before = 0, cnt = 0, bucket = nb - 1;
    for (long long b0 = 0; b0 < nb; b0 += 32) {
      const long long c = b0 + lane < nb ? h[b0 + lane] : 0;
      long long s = c;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const long long o = __shfl_up_sync(0xffffffffu, s, d);
        if (lane >= d) s += o;
      }
      const long long tot = __shfl_sync(0xffffffffu, s, 31);
      if (before + tot > r) {
        const int f = __ffs(__ballot_sync(0xffffffffu, before + s > r)) - 1;
        const long long sf = __shfl_sync(0xffffffffu, s, f), cf = __shfl_sync(0xffffffffu, c, f);
        bucket = b0 + f;
        r -= before + sf - cf;
        cnt = cf;
        break;
      }
      before += tot;
    }
    if (lane == 0) {
      const unsigned long long key = (A.pass == 0 ? 0ull : A.S.key[tk]) | ((unsigned long long)bucket << A.shift);
      A.S.key[tk] = key;
      A.S.rank[tk] = r;
      int j = 0;
      while (j < n_new && A.S.slot_key[seg * K + j] != key) ++j;
      if (j == n_new) {
        A.S.slot_key[seg * K + j] = key;
        ++n_new;
        matched += cnt;
      }
      A.S.slot[tk] = j;
    }
  }
  if (lane == 0) {
    A.S.n_slots[seg] = n_new;
    A.S.matched[seg] = matched;
  }
}

// ---- row form -------------------------------------------------------------------------------------------------------------
struct SelRowArgs {
  SelectPlan P;
  const long long* table;
  bool skip_nan;
  unsigned long long* keys;
  long long* nans;
};

template <class T>
__global__ void __launch_bounds__(kQThreads) select_row_kernel(const __grid_constant__ SelRowArgs A) {
  using KT = typename std::conditional<sizeof(T) == 8, unsigned long long, unsigned>::type;
  constexpr int BITS = 8 * sizeof(T);
  extern __shared__ __align__(16) unsigned char q_smem[];
  unsigned* hist = reinterpret_cast<unsigned*>(q_smem);
  KT* keys = reinterpret_cast<KT*>(q_smem + kQRowHist);
  __shared__ long long s_r;
  __shared__ KT s_prefix;
  __shared__ unsigned long long s_nan;
  const SelectPlan& P = A.P;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const long long seg = blockIdx.x, L = P.L, K = P.K, base = seg * L;
  if (t == 0) s_nan = 0;
  __syncthreads();
  unsigned nan = 0;
  for (long long i = t; i < L; i += kQThreads) {
    const KT k = (KT)s_key(s_load<T>(P.src, base + i));
    keys[i] = k;
    nan += k == (KT)s_nan_key<T>();
  }
  if (std::is_floating_point<T>::value) {
    for (int d = 16; d > 0; d >>= 1) nan += __shfl_xor_sync(0xffffffffu, nan, d);
    if (lane == 0 && nan) atomicAdd(&s_nan, (unsigned long long)nan);
  }
  __syncthreads();
  const long long nv = L - (long long)s_nan;
  const long long* ranks = A.table + (A.skip_nan ? nv * K : 0);
  long long prev_r = -1;
  KT prev_key = 0;
  for (long long k = 0; k < K; ++k) {
    const long long r0 = ranks[k];
    if (r0 == prev_r) {
      if (t == 0) A.keys[seg * K + k] = prev_key;
      continue;
    }
    long long r = r0;
    KT prefix = 0;
#pragma unroll 1
    for (int pass = 0; pass < BITS / 8; ++pass) {
      const int shift = BITS - 8 * (pass + 1);
      const KT mask = pass == 0 ? (KT)0 : (KT)(~(KT)0 << (shift + 8));
      hist[t] = 0u;  // (kQThreads == 256 counters)
      __syncthreads();
      for (long long i0 = (long long)warp * 32; i0 < L; i0 += kQThreads) {
        const long long i = i0 + lane;
        unsigned bin = kNone;
        if (i < L) {
          const KT kk = keys[i];
          if ((kk & mask) == prefix) bin = (unsigned)((kk >> shift) & 255u);
        }
        const unsigned add = warp_bin_share(bin, lane);
        if (add) atomicAdd(hist + bin, add);
      }
      __syncthreads();
      if (warp == 0) {
        unsigned c[8];
        long long s = 0;
#pragma unroll
        for (int v = 0; v < 8; ++v) {
          c[v] = hist[lane * 8 + v];
          s += c[v];
        }
        long long incl = s;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const long long o = __shfl_up_sync(0xffffffffu, incl, d);
          if (lane >= d) incl += o;
        }
        long long cum = incl - s;
        if (cum <= r && r < incl) {
#pragma unroll
          for (int v = 0; v < 8; ++v) {
            if (r < cum + c[v]) {
              s_r = r - cum;
              s_prefix = prefix | ((KT)(lane * 8 + v) << shift);
              break;
            }
            cum += c[v];
          }
        }
      }
      __syncthreads();
      r = s_r;
      prefix = s_prefix;
    }
    if (t == 0) A.keys[seg * K + k] = (unsigned long long)prefix;
    prev_r = r0;
    prev_key = prefix;
  }
  if (t == 0) A.nans[seg] = (long long)s_nan;
}

// ---- host: plans and dispatch --------------------------------------------------------------------------------------------
static long long q_cdiv(long long a, long long b) { return (a + b - 1) / b; }

const char* select_form_name(int form) { return form == SELECT_ROW ? "row" : "pass"; }

void make_select_plan(const rb200_index_view& src, int src_dtype, long long seg_len, long long targets, long long segments, bool no_row,
                      SelectPlan* P) {
  SelectPlan& p = *P;
  p = SelectPlan();
  p.src = make_compact_view(src);
  p.src_dtype = src_dtype;
  p.bits = src_dtype == RB200_F64 || src_dtype == RB200_I64 ? 64 : 32;
  const int kb = p.bits / 8, E = 16 / kb;
  p.n = 1;
  for (int d = 0; d < src.ndim; ++d) p.n *= src.shape[d];
  p.L = seg_len;
  p.S = p.n / seg_len;
  p.GS = segments > 0 ? segments : p.S;
  p.K = targets;
  const long long row_bytes = kQRowHist + seg_len * kb;
  p.form = segments == 0 && !no_row && row_bytes <= kQShared ? SELECT_ROW : SELECT_PASS;
  p.vec = p.src.nd == 1 && p.src.stride[0] == 1 && (((unsigned long long)p.src.base) & 15) == 0 && (p.S <= 1 || seg_len % E == 0);
  if (p.form == SELECT_ROW) {
    p.digit = 8;
    p.passes = p.bits / 8;
    p.chunk = seg_len;
    p.cps = 1;
    p.ctas = p.S;
    p.rows = targets;
    p.groups = 1;
    p.shared_bytes = row_bytes;
    return;
  }
  p.digit = p.GS == 1 && targets <= 12 ? 11 : 8;
  const long long nb = 1ll << p.digit;
  p.passes = (int)q_cdiv(p.bits, p.digit);
  p.rows = std::min(targets, kQShared / (nb * 4));
  p.groups = q_cdiv(targets, p.rows);
  p.cps = p.S ? std::max(1ll, std::min(q_cdiv(seg_len, kQUnit), q_cdiv(kQMaxCtas, p.S))) : 0;
  p.chunk = p.S ? q_cdiv(q_cdiv(seg_len, p.cps), kQUnit) * kQUnit : 0;
  p.cps = p.S ? q_cdiv(seg_len, p.chunk) : 0;
  p.ctas = p.S * p.cps;
  p.shared_bytes = p.rows * nb * 4;
  p.counts_bytes = p.GS * targets * nb * 8;
  p.cand_cap = p.GS == 1 ? std::min(p.n, std::max(p.n / 32, 65536ll)) : 0;
}

// pass p covers key bits [shift, hi)
static void sel_pass_bits(const SelectPlan& P, int pass, int* shift, int* width, unsigned long long* mask) {
  const int hi = P.bits - pass * P.digit;
  *shift = std::max(hi - P.digit, 0);
  *width = hi - *shift;
  *mask = pass == 0 ? 0ull : (~0ull << hi);
}

template <class T, int MODE> static cudaError_t sel_count_t(const SelCountArgs& A, unsigned grid, cudaStream_t s) {
  const auto k = select_count_kernel<T, MODE>;
  if (const cudaError_t e = allow_shared(k, A.P.shared_bytes)) return e;
  k<<<grid, kQThreads, (size_t)A.P.shared_bytes, s>>>(A);
  return cudaGetLastError();
}

template <class T> static cudaError_t sel_count_mode(const SelCountArgs& A, int mode, unsigned grid, cudaStream_t s) {
  if (mode == RB200_SELECT_APPEND) return sel_count_t<T, RB200_SELECT_APPEND>(A, grid, s);
  if (mode == RB200_SELECT_CAND) return sel_count_t<unsigned long long, RB200_SELECT_CAND>(A, grid, s);
  return sel_count_t<T, RB200_SELECT_READ>(A, grid, s);
}

cudaError_t launch_select_count(const SelectPlan& P, const rb200_select_state& S, int pass, int mode, cudaStream_t s) {
  if (P.GS == 0) return cudaSuccess;
  if (const cudaError_t e = cudaMemsetAsync(S.counts, 0, (size_t)P.counts_bytes, s)) return e;
  const bool fl = P.src_dtype == RB200_F64 || P.src_dtype == RB200_F32;
  if (pass == 0)
    if (const cudaError_t e = cudaMemsetAsync(S.nans, 0, (size_t)P.GS * 8, s)) return e;
  if (P.S == 0 || P.n == 0) return cudaSuccess;
  SelCountArgs A;
  A.P = P;
  A.S = S;
  A.pass = pass;
  sel_pass_bits(P, pass, &A.shift, &A.width, &A.mask);
  A.count_nan = pass == 0 && fl && mode != RB200_SELECT_CAND;
  long long grid = P.ctas;
  A.cchunk = 0;
  if (mode == RB200_SELECT_CAND) {
    grid = std::max(1ll, std::min(q_cdiv((long long)S.cand_cap, kQUnit), kQMaxCtas));
    A.cchunk = q_cdiv(q_cdiv(std::max((long long)S.cand_cap, 1ll), grid), kQUnit) * kQUnit;
  }
  for (long long g = 0; g < P.groups; ++g) {
    A.j0 = g * P.rows;
    cudaError_t e;
    switch (P.src_dtype) {
      case RB200_F64: e = sel_count_mode<double>(A, mode, (unsigned)grid, s); break;
      case RB200_F32: e = sel_count_mode<float>(A, mode, (unsigned)grid, s); break;
      case RB200_I64: e = sel_count_mode<long long>(A, mode, (unsigned)grid, s); break;
      default: e = sel_count_mode<int>(A, mode, (unsigned)grid, s); break;
    }
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t launch_select_choose(const SelectPlan& P, const rb200_select_state& S, int pass, cudaStream_t s) {
  if (P.GS == 0) return cudaSuccess;
  SelChooseArgs A;
  A.S = S;
  A.pass = pass;
  A.digit = P.digit;
  unsigned long long mask;
  sel_pass_bits(P, pass, &A.shift, &A.width, &mask);
  select_choose_kernel<<<(unsigned)q_cdiv(P.GS, kQChooseWarps), kQChooseWarps * 32, 0, s>>>(A);
  return cudaGetLastError();
}

template <class T> static cudaError_t sel_rows_t(const SelRowArgs& A, cudaStream_t s) {
  const auto k = select_row_kernel<T>;
  if (const cudaError_t e = allow_shared(k, A.P.shared_bytes)) return e;
  k<<<(unsigned)A.P.ctas, kQThreads, (size_t)A.P.shared_bytes, s>>>(A);
  return cudaGetLastError();
}

cudaError_t launch_select_rows(const SelectPlan& P, const long long* rank_table, bool skip_nan, unsigned long long* keys, long long* nans,
                               cudaStream_t s) {
  if (P.S == 0) return cudaSuccess;
  SelRowArgs A;
  A.P = P;
  A.table = rank_table;
  A.skip_nan = skip_nan;
  A.keys = keys;
  A.nans = nans;
  switch (P.src_dtype) {
    case RB200_F64: return sel_rows_t<double>(A, s);
    case RB200_F32: return sel_rows_t<float>(A, s);
    case RB200_I64: return sel_rows_t<long long>(A, s);
    default: return sel_rows_t<int>(A, s);
  }
}

}  // namespace rb200
