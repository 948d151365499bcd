// rb200_scan.cu — inclusive cumulative scans (cumsum / scumulative) in ONE pass over HBM (sm_90a).
//
// What it stands for in the reference: RemoteState.scumulative_worker (ramba/ramba.py:3378-3437) - every worker scans
// its part sequentially with the user's local function, then the boundary values are passed from worker to worker and
// folded in with the final function - behind cumsum (ramba/ramba.py:9675-9679) and scumulative (10057-10116).
//
// Here one rank's block is [outer][len][inner] (C order, the scan runs along `len`):
//   * inner == 1 (the scan axis is the fastest one): single-pass chained scan with decoupled look-back.  A tile is 2048
//     consecutive elements of one sequence (256 threads x 8); tiles are handed out in order by an atomic ticket, so a
//     tile only ever waits for tiles that are already running; a tile publishes its aggregate, looks back over its
//     predecessors with one warp (32 tiles per step) until it meets an inclusive prefix, then publishes its own.
//     Every element is read once and written once.
//   * inner > 1: one thread per (outer, inner) column walks `len` sequentially; consecutive threads own consecutive
//     `inner` indices, so every step of a warp is one coalesced row segment.  Also one read + one write per element.
// Accumulation class: float64 for float data (rounded to the dtype on store), int64 for integer data.  carry_in (one
// value per sequence / column, accumulator class) seeds the scan - the sum of the blocks that precede this rank's block
// along the axis; totals_out receives each sequence's total for the ranks that follow.
#include <cuda_runtime.h>
#include <stdio.h>

#include <string>

#include "rb200_launch.h"

namespace rb200 {

constexpr int kScanV = 8;
constexpr int kScanTile = kScanV * kThreads;

template <class A> __device__ __forceinline__ A scan_identity(int op);
// -0.0 for a float sum: -0.0 + x is x for every x, so a run of -0.0 scans to -0.0 (NumPy's cumsum), where +0.0 would not
template <> __device__ __forceinline__ double scan_identity<double>(int op) {
  return op == RB200_RED_ADD ? -0.0 : CT<double>::get(red_identity_bits(op, RB200_T_F64));
}
template <> __device__ __forceinline__ long long scan_identity<long long>(int op) { return (long long)red_identity_bits(op, RB200_T_I64); }

template <class A> __device__ __forceinline__ A shfl_up_a(A v, int d);
template <> __device__ __forceinline__ double shfl_up_a<double>(double v, int d) { return __shfl_up_sync(0xffffffffu, v, d); }
template <> __device__ __forceinline__ long long shfl_up_a<long long>(long long v, int d) { return __shfl_up_sync(0xffffffffu, v, d); }
template <class A> __device__ __forceinline__ A shfl_idx_a(A v, int l);
template <> __device__ __forceinline__ double shfl_idx_a<double>(double v, int l) { return __shfl_sync(0xffffffffu, v, l); }
template <> __device__ __forceinline__ long long shfl_idx_a<long long>(long long v, int l) { return __shfl_sync(0xffffffffu, v, l); }

struct ScanScratch {
  unsigned int* ticket;
  volatile int* flag;  // 0: nothing yet, 1: aggregate published, 2: inclusive prefix published
  volatile unsigned long long* agg;
  volatile unsigned long long* incl;
};

template <class A> __device__ __forceinline__ unsigned long long a_bits(A v);
template <> __device__ __forceinline__ unsigned long long a_bits<double>(double v) { return (unsigned long long)__double_as_longlong(v); }
template <> __device__ __forceinline__ unsigned long long a_bits<long long>(long long v) { return (unsigned long long)v; }
template <class A> __device__ __forceinline__ A a_from(unsigned long long b);
template <> __device__ __forceinline__ double a_from<double>(unsigned long long b) { return __longlong_as_double((long long)b); }
template <> __device__ __forceinline__ long long a_from<long long>(unsigned long long b) { return (long long)b; }

// S: storage type, A: accumulator type
template <class S, class A>
__global__ void __launch_bounds__(kThreads) scan_lookback_kernel(const S* __restrict__ src, S* __restrict__ dst, long long n_seq, long long len,
                                                                  long long tiles_per_seq, int op, const A* __restrict__ carry_in, A* __restrict__ totals_out,
                                                                  ScanScratch sc) {
  __shared__ A warp_tot[kThreads / 32];
  __shared__ long long s_tile;
  __shared__ A s_prefix;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long n_tiles = n_seq * tiles_per_seq;
  const A ident = scan_identity<A>(op);
  for (;;) {
    if (tid == 0) s_tile = (long long)atomicAdd(sc.ticket, 1u);
    __syncthreads();
    const long long t = s_tile;
    if (t >= n_tiles) return;
    const long long seq = t / tiles_per_seq, j = t - seq * tiles_per_seq;
    const long long e0 = j * kScanTile + (long long)tid * kScanV;  // first element of this thread inside the sequence
    const S* sp = src + seq * len + e0;
    A x[kScanV];
#pragma unroll
    for (int k = 0; k < kScanV; ++k) x[k] = (e0 + k < len) ? (A)sp[k] : ident;
    // thread-local inclusive scan, then the thread totals across the warp and the CTA
#pragma unroll
    for (int k = 1; k < kScanV; ++k) x[k] = red_combine<A>(op, x[k - 1], x[k]);
    A tot = x[kScanV - 1];
    A inc = tot;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const A o = shfl_up_a<A>(inc, d);
      if (lane >= d) inc = red_combine<A>(op, o, inc);
    }
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    A before = ident;  // everything in this tile before this thread
    A tile_agg = ident;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
      const A wt = warp_tot[w];
      if (w < warp) before = red_combine<A>(op, before, wt);
      tile_agg = red_combine<A>(op, tile_agg, wt);
    }
    const A excl_in_warp = shfl_up_a<A>(inc, 1);
    if (lane > 0) before = red_combine<A>(op, before, excl_in_warp);

    // ---- decoupled look-back (warp 0): exclusive prefix of this tile within its sequence
    if (warp == 0) {
      const long long first = seq * tiles_per_seq;
      A prefix = carry_in ? carry_in[seq] : ident;
      if (j > 0) {
        if (lane == 0) {
          sc.agg[t] = a_bits<A>(tile_agg);
          __threadfence();
          sc.flag[t] = 1;
        }
        A run = ident;
        long long base = t - 1;
        for (;;) {
          const long long p = base - lane;
          int st = 2;
          A v = ident;
          if (p >= first) {
            do {
              st = sc.flag[p];
            } while (st == 0);
            __threadfence();
            v = a_from<A>(st == 2 ? sc.incl[p] : sc.agg[p]);
          }
          const unsigned done = __ballot_sync(0xffffffffu, st == 2);
          const int stop = done ? (__ffs(done) - 1) : 31;  // closest tile that already has an inclusive prefix
          if (lane > stop) v = ident;
          // combine lanes 0..stop, closest tile first (the operations are commutative; order only affects fp rounding)
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) {
            const A o = shfl_idx_a<A>(v, (lane + d) & 31);
            if (lane + d < 32) v = red_combine<A>(op, v, o);
          }
          run = red_combine<A>(op, shfl_idx_a<A>(v, 0), run);
          if (done) break;
          base -= 32;
        }
        prefix = red_combine<A>(op, prefix, run);
      }
      if (lane == 0) {
        sc.incl[t] = a_bits<A>(red_combine<A>(op, prefix, tile_agg));
        __threadfence();
        sc.flag[t] = 2;
        s_prefix = prefix;
        if (totals_out && j == tiles_per_seq - 1) totals_out[seq] = red_combine<A>(op, prefix, tile_agg);
      }
    }
    __syncthreads();
    const A base_v = red_combine<A>(op, s_prefix, before);
    S* dp = dst + seq * len + e0;
#pragma unroll
    for (int k = 0; k < kScanV; ++k)
      if (e0 + k < len) dp[k] = (S)red_combine<A>(op, base_v, x[k]);
    __syncthreads();
  }
}

template <class S, class A>
__global__ void __launch_bounds__(kThreads) scan_columns_kernel(const S* __restrict__ src, S* __restrict__ dst, long long n_outer, long long len,
                                                                 long long n_inner, int op, const A* __restrict__ carry_in, A* __restrict__ totals_out) {
  const long long n_cols = n_outer * n_inner;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < n_cols; c += (long long)gridDim.x * blockDim.x) {
    const long long o = c / n_inner, i = c - o * n_inner;
    const S* sp = src + o * len * n_inner + i;
    S* dp = dst + o * len * n_inner + i;
    A acc = carry_in ? carry_in[c] : scan_identity<A>(op);
#pragma unroll 8
    for (long long l = 0; l < len; ++l) {
      acc = red_combine<A>(op, acc, (A)sp[l * n_inner]);
      dp[l * n_inner] = (S)acc;
    }
    if (totals_out) totals_out[c] = acc;
  }
}

template <class S, class A>
static cudaError_t scan_launch(const void* src, void* dst, long long n_outer, long long len, long long n_inner, int op, const void* carry, void* totals,
                               void* scratch, int sms, cudaStream_t stream) {
  if (n_inner == 1) {
    const long long tiles_per_seq = (len + kScanTile - 1) / kScanTile;
    const long long n_tiles = n_outer * tiles_per_seq;
    // scratch layout: [ticket 256 B][flag int * n_tiles, padded to 8][agg u64 * n_tiles][incl u64 * n_tiles]
    const size_t flag_bytes = ((size_t)n_tiles * 4 + 255) / 256 * 256;
    cudaError_t e = cudaMemsetAsync(scratch, 0, 256 + flag_bytes, stream);
    if (e != cudaSuccess) return e;
    ScanScratch sc;
    sc.ticket = (unsigned int*)scratch;
    sc.flag = (volatile int*)((char*)scratch + 256);
    sc.agg = (volatile unsigned long long*)((char*)scratch + 256 + flag_bytes);
    sc.incl = sc.agg + n_tiles;
    long long blocks = n_tiles < (long long)sms * 4 ? n_tiles : (long long)sms * 4;
    scan_lookback_kernel<S, A><<<(unsigned)blocks, kThreads, 0, stream>>>((const S*)src, (S*)dst, n_outer, len, tiles_per_seq, op, (const A*)carry, (A*)totals, sc);
  } else {
    const long long n_cols = n_outer * n_inner;
    long long blocks = (n_cols + kThreads - 1) / kThreads;
    if (blocks > (long long)sms * 8) blocks = (long long)sms * 8;
    scan_columns_kernel<S, A><<<(unsigned)blocks, kThreads, 0, stream>>>((const S*)src, (S*)dst, n_outer, len, n_inner, op, (const A*)carry, (A*)totals);
  }
  return cudaGetLastError();
}

long long scan_scratch_bytes(long long n_outer, long long len, long long n_inner) {
  if (n_inner != 1) return 256;
  const long long n_tiles = n_outer * ((len + kScanTile - 1) / kScanTile);
  const long long flag_bytes = (n_tiles * 4 + 255) / 256 * 256;
  return 256 + flag_bytes + 16 * n_tiles + 256;
}

cudaError_t launch_scan(const void* src, void* dst, int dtype, long long n_outer, long long len, long long n_inner, int op, const void* carry, void* totals,
                        void* scratch, int sms, cudaStream_t stream, bool* supported) {
  *supported = true;
  switch (dtype) {
    case RB200_F64: return scan_launch<double, double>(src, dst, n_outer, len, n_inner, op, carry, totals, scratch, sms, stream);
    case RB200_F32: return scan_launch<float, double>(src, dst, n_outer, len, n_inner, op, carry, totals, scratch, sms, stream);
    case RB200_I64: return scan_launch<long long, long long>(src, dst, n_outer, len, n_inner, op, carry, totals, scratch, sms, stream);
    case RB200_I32: return scan_launch<int, long long>(src, dst, n_outer, len, n_inner, op, carry, totals, scratch, sms, stream);
    default: *supported = false; return cudaSuccess;
  }
}

}  // namespace rb200
