// rb200_index.cu — integer-array indexing on sm_90a: gather, scatter and the route step of the multi-rank exchange.
//
// What it stands for in the reference: getitem_array_executor / setitem_array_executor (ramba/ramba.py:6429-6545,
// 6143-6297) move one element at a time in Python on the workers.  Here the host hands over `lin`, the C-order linear
// index of every addressed element within a view, and these kernels move the elements:
//   * gather / scatter: a persistent grid; each thread takes 4 consecutive entries of lin with two 16-byte loads, reads or
//     writes the 4 addressed elements and stores or loads the 4 contiguous ones as one vector when aligned.  A 1-D view
//     (after the host collapsed contiguous dims) costs one multiply per element; an N-d view decodes lin with 32-bit
//     divisions when the view has fewer than 2^32 elements and with 64-bit ones otherwise.  Addresses are 64-bit.
//   * route: three launches.  Warp w owns a tile of kRouteTile consecutive requests.  (1) count the requests of each owner
//     in every tile; (2) one CTA per owner scans its column of tile counts; (3) every warp walks its tile again in order,
//     32 requests at a time, and places each request after the earlier ones of the same owner (__match_any_sync).  The
//     grouping therefore depends only on the input.
// Out-of-range entries are counted with one atomic per warp (__reduce_add_sync) and never dereferenced.
#include <cuda_runtime.h>

#include "rb200_index.h"

namespace rb200 {

constexpr int kIdxThreads = 256;
constexpr int kIdxV = 4;  // entries of lin per thread per step
constexpr int kRouteWarps = kIdxThreads / 32;
constexpr int kRouteTile = 32 * 64;  // requests per warp tile

template <int B> struct ElemT;
template <> struct ElemT<1> { using T = unsigned char; };
template <> struct ElemT<2> { using T = unsigned short; };
template <> struct ElemT<4> { using T = unsigned int; };
template <> struct ElemT<8> { using T = unsigned long long; };

template <class T> struct alignas(sizeof(T) * kIdxV) Vec { T v[kIdxV]; };

enum { MODE_FLAT = 0, MODE_ND32 = 1, MODE_ND64 = 2 };

// element offset of linear index l (0 <= l < size) in view v
template <int MODE> __device__ __forceinline__ long long elem_offset(const IdxView& v, long long l) {
  if (MODE == MODE_FLAT) return l * v.stride[0];
  long long off = 0;
  if (MODE == MODE_ND32) {
    unsigned r = (unsigned)l;
#pragma unroll
    for (int d = RB200_MAX_DIMS - 1; d > 0; --d) {
      if (d < v.ndim) {
        const unsigned e = (unsigned)v.shape[d];
        const unsigned q = r / e;
        off += (long long)(r - q * e) * v.stride[d];
        r = q;
      }
    }
    return off + (long long)r * v.stride[0];
  }
  long long r = l;
#pragma unroll
  for (int d = RB200_MAX_DIMS - 1; d > 0; --d) {
    if (d < v.ndim) {
      const long long e = v.shape[d];
      const long long q = r / e;
      off += (r - q * e) * v.stride[d];
      r = q;
    }
  }
  return off + r * v.stride[0];
}

__device__ __forceinline__ bool in_range(long long l, long long size) { return (unsigned long long)l < (unsigned long long)size; }

__device__ __forceinline__ void count_bad(unsigned nbad, unsigned long long* bad) {
  nbad = __reduce_add_sync(0xffffffffu, nbad);
  if ((threadIdx.x & 31) == 0 && nbad) atomicAdd(bad, (unsigned long long)nbad);
}

// VEC: lin is 16-byte aligned and out is aligned to kIdxV elements
template <int B, int MODE, bool VEC>
__global__ void __launch_bounds__(kIdxThreads) gather_kernel(IdxView v, const long long* __restrict__ lin, long long n,
                                                             typename ElemT<B>::T* __restrict__ out, unsigned long long* bad) {
  using T = typename ElemT<B>::T;
  const T* __restrict__ base = (const T*)v.base;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nth = (long long)gridDim.x * blockDim.x;
  unsigned nbad = 0;
  long long i0 = 0;
  if (VEC) {
    const long long nv = n / kIdxV;
    for (long long j = tid; j < nv; j += nth) {
      const longlong2* p = reinterpret_cast<const longlong2*>(lin + j * kIdxV);
      const longlong2 a = __ldcs(p), b = __ldcs(p + 1);
      const long long l[kIdxV] = {a.x, a.y, b.x, b.y};
      Vec<T> o;
#pragma unroll
      for (int k = 0; k < kIdxV; ++k) {
        const bool ok = in_range(l[k], v.size);
        o.v[k] = ok ? base[elem_offset<MODE>(v, l[k])] : T(0);
        nbad += ok ? 0u : 1u;
      }
      *reinterpret_cast<Vec<T>*>(out + j * kIdxV) = o;
    }
    i0 = nv * kIdxV;
  }
  for (long long i = i0 + tid; i < n; i += nth) {
    const long long l = lin[i];
    const bool ok = in_range(l, v.size);
    out[i] = ok ? base[elem_offset<MODE>(v, l)] : T(0);
    nbad += ok ? 0u : 1u;
  }
  count_bad(nbad, bad);
}

template <int B, int MODE, bool VEC>
__global__ void __launch_bounds__(kIdxThreads) scatter_kernel(IdxView v, const long long* __restrict__ lin, long long n,
                                                              const typename ElemT<B>::T* __restrict__ values, unsigned long long* bad) {
  using T = typename ElemT<B>::T;
  T* base = (T*)v.base;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nth = (long long)gridDim.x * blockDim.x;
  unsigned nbad = 0;
  long long i0 = 0;
  if (VEC) {
    const long long nv = n / kIdxV;
    for (long long j = tid; j < nv; j += nth) {
      const longlong2* p = reinterpret_cast<const longlong2*>(lin + j * kIdxV);
      const longlong2 a = __ldcs(p), b = __ldcs(p + 1);
      const long long l[kIdxV] = {a.x, a.y, b.x, b.y};
      const Vec<T> x = *reinterpret_cast<const Vec<T>*>(values + j * kIdxV);
#pragma unroll
      for (int k = 0; k < kIdxV; ++k) {
        if (in_range(l[k], v.size))
          base[elem_offset<MODE>(v, l[k])] = x.v[k];
        else
          ++nbad;
      }
    }
    i0 = nv * kIdxV;
  }
  for (long long i = i0 + tid; i < n; i += nth) {
    const long long l = lin[i];
    if (in_range(l, v.size))
      base[elem_offset<MODE>(v, l)] = values[i];
    else
      ++nbad;
  }
  count_bad(nbad, bad);
}

// ---- host: view collapse and dispatch -------------------------------------------------------------------------------
IdxView collapse_index_view(const rb200_index_view& in) {
  IdxView v;
  v.base = (char*)in.base;
  v.elem_bytes = in.elem_bytes;
  v.size = 1;
  for (int d = 0; d < in.ndim; ++d) v.size *= in.shape[d];
  int k = 0;
  for (int d = 0; d < in.ndim; ++d) {
    if (in.shape[d] == 1) continue;
    if (k > 0 && v.stride[k - 1] == in.stride[d] * in.shape[d]) {  // contiguous with the previous kept dim: merge
      v.shape[k - 1] *= in.shape[d];
      v.stride[k - 1] = in.stride[d];
      continue;
    }
    v.shape[k] = in.shape[d];
    v.stride[k] = in.stride[d];
    ++k;
  }
  if (k == 0 || v.size == 0) {  // one element, or none (every entry is then out of range)
    v.shape[0] = v.size;
    v.stride[0] = 1;
    k = 1;
  }
  v.ndim = k;
  return v;
}

static unsigned idx_blocks(long long n, int sms) {
  long long b = (n + (long long)kIdxThreads * kIdxV - 1) / ((long long)kIdxThreads * kIdxV);
  if (b > (long long)sms * 8) b = (long long)sms * 8;
  return (unsigned)(b < 1 ? 1 : b);
}

static int idx_mode(const IdxView& v) { return v.ndim == 1 ? MODE_FLAT : v.size <= 0xffffffffLL ? MODE_ND32 : MODE_ND64; }

template <int B, int MODE>
static void gather_vec(bool vec, const IdxView& v, const long long* lin, long long n, void* out, unsigned long long* bad, unsigned blocks,
                       cudaStream_t s) {
  using T = typename ElemT<B>::T;
  if (vec)
    gather_kernel<B, MODE, true><<<blocks, kIdxThreads, 0, s>>>(v, lin, n, (T*)out, bad);
  else
    gather_kernel<B, MODE, false><<<blocks, kIdxThreads, 0, s>>>(v, lin, n, (T*)out, bad);
}

template <int B>
static void gather_b(int mode, bool vec, const IdxView& v, const long long* lin, long long n, void* out, unsigned long long* bad,
                     unsigned blocks, cudaStream_t s) {
  if (mode == MODE_FLAT) gather_vec<B, MODE_FLAT>(vec, v, lin, n, out, bad, blocks, s);
  else if (mode == MODE_ND32) gather_vec<B, MODE_ND32>(vec, v, lin, n, out, bad, blocks, s);
  else gather_vec<B, MODE_ND64>(vec, v, lin, n, out, bad, blocks, s);
}

template <int B, int MODE>
static void scatter_vec(bool vec, const IdxView& v, const long long* lin, long long n, const void* values, unsigned long long* bad,
                        unsigned blocks, cudaStream_t s) {
  using T = typename ElemT<B>::T;
  if (vec)
    scatter_kernel<B, MODE, true><<<blocks, kIdxThreads, 0, s>>>(v, lin, n, (const T*)values, bad);
  else
    scatter_kernel<B, MODE, false><<<blocks, kIdxThreads, 0, s>>>(v, lin, n, (const T*)values, bad);
}

template <int B>
static void scatter_b(int mode, bool vec, const IdxView& v, const long long* lin, long long n, const void* values, unsigned long long* bad,
                      unsigned blocks, cudaStream_t s) {
  if (mode == MODE_FLAT) scatter_vec<B, MODE_FLAT>(vec, v, lin, n, values, bad, blocks, s);
  else if (mode == MODE_ND32) scatter_vec<B, MODE_ND32>(vec, v, lin, n, values, bad, blocks, s);
  else scatter_vec<B, MODE_ND64>(vec, v, lin, n, values, bad, blocks, s);
}

static bool aligned(const void* p, size_t a) { return ((size_t)p & (a - 1)) == 0; }

cudaError_t launch_gather(const IdxView& v, const long long* lin, long long n, void* out, unsigned long long* bad, int sms, cudaStream_t s) {
  const bool vec = aligned(lin, 16) && aligned(out, (size_t)v.elem_bytes * kIdxV);
  const unsigned blocks = idx_blocks(n, sms);
  const int mode = idx_mode(v);
  switch (v.elem_bytes) {
    case 1: gather_b<1>(mode, vec, v, lin, n, out, bad, blocks, s); break;
    case 2: gather_b<2>(mode, vec, v, lin, n, out, bad, blocks, s); break;
    case 4: gather_b<4>(mode, vec, v, lin, n, out, bad, blocks, s); break;
    default: gather_b<8>(mode, vec, v, lin, n, out, bad, blocks, s); break;
  }
  return cudaGetLastError();
}

cudaError_t launch_scatter(const IdxView& v, const long long* lin, long long n, const void* values, unsigned long long* bad, int sms,
                           cudaStream_t s) {
  const bool vec = aligned(lin, 16) && aligned(values, (size_t)v.elem_bytes * kIdxV);
  const unsigned blocks = idx_blocks(n, sms);
  const int mode = idx_mode(v);
  switch (v.elem_bytes) {
    case 1: scatter_b<1>(mode, vec, v, lin, n, values, bad, blocks, s); break;
    case 2: scatter_b<2>(mode, vec, v, lin, n, values, bad, blocks, s); break;
    case 4: scatter_b<4>(mode, vec, v, lin, n, values, bad, blocks, s); break;
    default: scatter_b<8>(mode, vec, v, lin, n, values, bad, blocks, s); break;
  }
  return cudaGetLastError();
}

// ---- route ----------------------------------------------------------------------------------------------------------
// owner of linear index l of the routed view (-1: out of range) and its local element offset.  Two walks over the dims
// (the first finds the cell, the second needs the cell's strides) instead of per-dim arrays, which ptxas put on the stack.
__device__ __forceinline__ int locate(const RouteParams& R, long long l, long long* off) {
  if (!in_range(l, R.size)) return -1;
  int cell = 0, mult = 1;
  long long r = l;
#pragma unroll
  for (int d = RB200_MAX_DIMS - 1; d >= 0; --d) {
    if (d < R.ndim) {
      const long long q = r / R.shape[d];
      const long long c = r - q * R.shape[d];
      r = q;
      const long long* cut = R.cuts + R.cut_start[d];
      int j = 0;
      while (c >= cut[j + 1]) ++j;
      cell += j * mult;
      mult *= R.n_cells[d];
    }
  }
  long long o = R.offset[cell];
  r = l;
#pragma unroll
  for (int d = RB200_MAX_DIMS - 1; d >= 0; --d) {
    if (d < R.ndim) {
      const long long q = r / R.shape[d];
      const long long c = r - q * R.shape[d];
      r = q;
      const long long* cut = R.cuts + R.cut_start[d];
      int j = 0;
      while (c >= cut[j + 1]) ++j;
      o += (c - cut[j]) * R.stride[cell * R.ndim + d];
    }
  }
  *off = o;
  return R.owner[cell];
}

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// (1) tile_counts[t * n_ranks + r] = requests of tile t owned by rank r
__global__ void __launch_bounds__(kIdxThreads) route_count_kernel(const __grid_constant__ RouteParams R, const long long* __restrict__ lin,
                                                                  long long n, long long n_tiles, long long* tile_counts,
                                                                  unsigned long long* bad) {
  __shared__ int cnt[kRouteWarps][RB200_MAX_ROUTE_RANKS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned nbad = 0;
  const long long nwarps = (long long)gridDim.x * kRouteWarps;
  for (long long t = (long long)blockIdx.x * kRouteWarps + warp; t < n_tiles; t += nwarps) {
    for (int r = lane; r < R.n_ranks; r += 32) cnt[warp][r] = 0;
    __syncwarp();
    const long long i0 = t * kRouteTile;
    for (int s = 0; s < kRouteTile; s += 32) {
      const long long i = i0 + s + lane;
      int o = -2;  // past the end
      if (i < n) {
        long long off;
        o = locate(R, lin[i], &off);
        nbad += o < 0 ? 1u : 0u;
      }
      const unsigned same = __match_any_sync(0xffffffffu, o);
      if (o >= 0 && (same & lanemask_lt()) == 0) cnt[warp][o] += __popc(same);
      __syncwarp();
    }
    for (int r = lane; r < R.n_ranks; r += 32) tile_counts[t * R.n_ranks + r] = cnt[warp][r];
    __syncwarp();
  }
  count_bad(nbad, bad);
}

// (2) one CTA per rank r: exclusive scan of column r of tile_counts in place, counts[r] = its total
__global__ void __launch_bounds__(kIdxThreads) route_scan_kernel(long long* tile_counts, long long n_tiles, int n_ranks, long long* counts) {
  __shared__ long long wsum[kRouteWarps];
  const int r = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long run = 0;
  for (long long t0 = 0; t0 < n_tiles; t0 += kIdxThreads) {
    const long long t = t0 + threadIdx.x;
    const long long x = t < n_tiles ? tile_counts[t * n_ranks + r] : 0;
    long long inc = x;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += y;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    long long before = run, total = 0;
#pragma unroll
    for (int w = 0; w < kRouteWarps; ++w) {
      if (w < warp) before += wsum[w];
      total += wsum[w];
    }
    if (t < n_tiles) tile_counts[t * n_ranks + r] = before + inc - x;
    run += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[r] = run;
}

// (3) place every request of tile t after the earlier ones of the same owner
__global__ void __launch_bounds__(kIdxThreads) route_place_kernel(const __grid_constant__ RouteParams R, const long long* __restrict__ lin,
                                                                  long long n, long long n_tiles, const long long* __restrict__ tile_base,
                                                                  const long long* __restrict__ counts, long long* __restrict__ offsets,
                                                                  long long* __restrict__ slots) {
  __shared__ long long start[RB200_MAX_ROUTE_RANKS];
  __shared__ long long next[kRouteWarps][RB200_MAX_ROUTE_RANKS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    long long s = 0;
    for (int r = 0; r < R.n_ranks; ++r) {
      start[r] = s;
      s += counts[r];
    }
  }
  __syncthreads();
  const long long nwarps = (long long)gridDim.x * kRouteWarps;
  for (long long t = (long long)blockIdx.x * kRouteWarps + warp; t < n_tiles; t += nwarps) {
    for (int r = lane; r < R.n_ranks; r += 32) next[warp][r] = start[r] + tile_base[t * R.n_ranks + r];
    __syncwarp();
    const long long i0 = t * kRouteTile;
    for (int s = 0; s < kRouteTile; s += 32) {
      const long long i = i0 + s + lane;
      int o = -2;
      long long off = 0;
      if (i < n) o = locate(R, lin[i], &off);
      const unsigned same = __match_any_sync(0xffffffffu, o);
      if (o >= 0) {
        const long long slot = next[warp][o] + __popc(same & lanemask_lt());
        offsets[slot] = off;
        slots[i] = slot;
      } else if (o == -1) {
        slots[i] = -1;
      }
      __syncwarp();
      if (o >= 0 && (same & lanemask_lt()) == 0) next[warp][o] += __popc(same);
      __syncwarp();
    }
  }
}

static long long route_tiles(long long n) { return (n + kRouteTile - 1) / kRouteTile; }

long long route_scratch_bytes(long long n, int n_ranks) { return 256 + route_tiles(n) * (long long)n_ranks * 8; }

cudaError_t launch_route(const RouteParams& R, const long long* lin, long long n, long long* offsets, long long* slots, long long* counts,
                         unsigned long long* bad, void* scratch, int sms, cudaStream_t s) {
  const long long n_tiles = route_tiles(n);
  long long* tile_counts = (long long*)scratch;
  long long blocks = (n_tiles + kRouteWarps - 1) / kRouteWarps;
  if (blocks > (long long)sms * 4) blocks = (long long)sms * 4;
  if (blocks < 1) blocks = 1;
  route_count_kernel<<<(unsigned)blocks, kIdxThreads, 0, s>>>(R, lin, n, n_tiles, tile_counts, bad);
  route_scan_kernel<<<(unsigned)R.n_ranks, kIdxThreads, 0, s>>>(tile_counts, n_tiles, R.n_ranks, counts);
  route_place_kernel<<<(unsigned)blocks, kIdxThreads, 0, s>>>(R, lin, n, n_tiles, tile_counts, counts, offsets, slots);
  return cudaGetLastError();
}

}  // namespace rb200
