// rb200_hbm_probe.cu — probe kernels for the write-heavy HBM rate (benchmarks/hbm_mix.py).  Not part of the library:
// its own shared object (`make probe`), so nothing here reaches libramba_b200.so.
//
// Every kernel streams float64 `out_j = A * s_j` for j < n_out (1 or 3 outputs) with the layout of the library's 1-D
// kernels: 256 threads, tile = 2048 elements, element k of thread t at tile*2048 + k*256 + t.  A is staged by one bulk
// copy per full tile into a ring of `depth` stages (mbarrier completion, one CTA barrier per tile), as the lean
// interpreter and the streaming kernel do.  The arms vary how the results reach HBM (FORM), the tile walk (WALK), the
// read side (LOAD) and the grid:
//   FORM 0  plain: one 8-byte store per element (the library's form)
//   FORM 1  warp-pair shuffle: for each pair (k, k+1) even lanes store (x[k] of lane, lane+1), odd lanes the k+1 pair,
//           as 16-byte stores; the values are unchanged, half the store instructions
//   FORM 2  staged: each output's tile image is written to shared memory in [k][thread] order and leaves by one
//           cp.async.bulk (shared -> global) per output and tile; wait_group.read before the staging is rewritten
//   WALK 0  round-robin: CTA b walks tiles b, b+grid, ...      WALK 1  contiguous: CTA b owns one range of tiles
//   LOAD 1  (read side, plain stores only) no staging: each thread loads its 8 elements with 8-byte loads
// The grid is CTAs/SM x SMs, or one CTA per tile when 0 CTAs/SM are asked for.  The direct load form can also cap the
// CTAs resident per SM (`resident`, by padding the dynamic shared memory) and walk with CTAs/SM up to 8.  The ragged last tile is read directly
// and written with predicated 8-byte stores in every form.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../rb200_vm.cuh"

namespace rb200 {
namespace probe {

constexpr int V = 8;
constexpr int TILE = kThreads * V;
constexpr unsigned SLOT = TILE * 8u;

struct Args {
  const double* a;
  double* out[3];
  double s[3];
  long long n, n_tiles;
  int n_out, depth;
};

__device__ __forceinline__ void st_v2(double* p, double x, double y) {
  asm volatile("st.global.v2.f64 [%0], {%1, %2};" ::"l"(p), "d"(x), "d"(y) : "memory");
}

template <int FORM, int WALK, int MINB, int LOAD> __global__ void __launch_bounds__(kThreads, MINB) probe_kernel(const __grid_constant__ Args P) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) u64 mbar[8];
  const unsigned smem_s = (unsigned)__cvta_generic_to_shared(smem);
  const unsigned mbar_s = (unsigned)__cvta_generic_to_shared(mbar);
  const unsigned stage_s = smem_s + (unsigned)P.depth * SLOT;  // FORM 2: n_out staging slots behind the ring
  const unsigned tid = threadIdx.x, lane = tid & 31u;
  if (tid == 0) {
    for (int s = 0; s < P.depth; ++s) mbar_init(mbar_s + 8u * s, 1u);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  long long t0, t1, tstep;
  if (WALK == 0) {
    t0 = blockIdx.x;
    t1 = P.n_tiles;
    tstep = gridDim.x;
  } else {
    t0 = P.n_tiles * blockIdx.x / gridDim.x;
    t1 = P.n_tiles * (blockIdx.x + 1) / gridDim.x;
    tstep = 1;
  }
  const long long n_it = t1 > t0 ? (t1 - t0 + tstep - 1) / tstep : 0;
  auto full = [&](long long it) { return (t0 + it * tstep + 1) * TILE <= P.n; };
  auto issue = [&](long long it) {
    const unsigned slot = (unsigned)(it % P.depth);
    mbar_expect_tx(mbar_s + 8u * slot, SLOT);
    bulk_g2s(smem_s + slot * SLOT, P.a + (t0 + it * tstep) * TILE, SLOT, mbar_s + 8u * slot);
  };
  if (LOAD == 0 && tid == 0)
    for (long long it = 0; it < P.depth - 1 && it < n_it; ++it)
      if (full(it)) issue(it);
  for (long long it = 0; it < n_it; ++it) {
    const long long tile = t0 + it * tstep;
    const bool f = full(it);
    if (LOAD == 0) __syncthreads();
    if (LOAD == 0 && tid == 0) {
      const long long nx = it + P.depth - 1;
      if (nx < n_it && full(nx)) issue(nx);
    }
    double x[V];
    const long long e0 = tile * TILE + tid;
    if (LOAD == 0 && f) {
      const unsigned slot = (unsigned)(it % P.depth);
      mbar_wait(mbar_s + 8u * slot, (unsigned)((it / P.depth) & 1));
#pragma unroll
      for (int k = 0; k < V; ++k) x[k] = __longlong_as_double((long long)lds64(smem_s + slot * SLOT + (k * kThreads + tid) * 8u));
    } else {
#pragma unroll
      for (int k = 0; k < V; ++k) x[k] = e0 + k * kThreads < P.n ? ldg<double>(P.a + e0 + k * kThreads) : 0.0;
    }
    if (FORM == 2 && f) {
      // the previous tile's bulk stores have finished reading the staging slots
      if (tid == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      __syncthreads();
    }
#pragma unroll 1
    for (int j = 0; j < P.n_out; ++j) {
      double r[V];
#pragma unroll
      for (int k = 0; k < V; ++k) r[k] = __dmul_rn(x[k], P.s[j]);
      double* p = P.out[j] + e0;
      if (!f) {
#pragma unroll
        for (int k = 0; k < V; ++k)
          if (e0 + k * kThreads < P.n) stg<double>(p + k * kThreads, r[k]);
      } else if (FORM == 0) {
#pragma unroll
        for (int k = 0; k < V; ++k) stg<double>(p + k * kThreads, r[k]);
      } else if (FORM == 1) {
        const bool odd = lane & 1u;
        double* q = P.out[j] + tile * TILE + (tid & ~1u);
#pragma unroll
        for (int k = 0; k < V; k += 2) {
          const double give = odd ? r[k] : r[k + 1];
          const double got = __shfl_xor_sync(0xffffffffu, give, 1);
          if (odd) st_v2(q + (k + 1) * kThreads, got, r[k + 1]);
          else st_v2(q + k * kThreads, r[k], got);
        }
      } else {
        const unsigned dst = stage_s + (unsigned)j * SLOT + tid * 8u;
#pragma unroll
        for (int k = 0; k < V; ++k) sts64(dst + k * kThreads * 8u, (u64)__double_as_longlong(r[k]));
      }
    }
    if (FORM == 2 && f) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
      if (tid == 0) {
        for (int j = 0; j < P.n_out; ++j)
          asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(P.out[j] + tile * TILE), "r"(stage_s + (unsigned)j * SLOT), "r"(SLOT)
                       : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    }
  }
  if (FORM == 2 && tid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <int FORM, int WALK, int MINB, int LOAD = 0>
int launch(const Args& P, int sms, cudaStream_t st, bool per_tile = false, int grid_per_sm = MINB, int resident = 0) {
  size_t smem = (LOAD == 0 ? (size_t)P.depth * SLOT : 0) + (FORM == 2 ? (size_t)P.n_out * SLOT : 0);
  if (resident > 0) smem = (size_t)(200 * 1024) / resident;  // at most `resident` CTAs fit in 228 KB per SM
  cudaError_t e = cudaFuncSetAttribute(probe_kernel<FORM, WALK, MINB, LOAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, probe_kernel<FORM, WALK, MINB, LOAD>, kThreads, smem);
  if (e != cudaSuccess) return (int)e;
  if (per_sm < MINB) return -per_sm - 1;  // the form does not fit MINB CTAs per SM
  if (resident > 0 && per_sm > resident) return -100;
  long long blocks = per_tile ? P.n_tiles : (long long)sms * grid_per_sm;
  if (blocks > P.n_tiles) blocks = P.n_tiles;
  probe_kernel<FORM, WALK, MINB, LOAD><<<(unsigned)blocks, kThreads, smem, st>>>(P);
  return (int)cudaGetLastError();
}

template <int FORM, int WALK> int by_minb(const Args& P, int minb, int sms, cudaStream_t st) {
  switch (minb) {
    case 0: return launch<FORM, WALK, 2>(P, sms, st, true);
    case 1: return launch<FORM, WALK, 1>(P, sms, st);
    case 2: return launch<FORM, WALK, 2>(P, sms, st);
    case 3: return launch<FORM, WALK, 3>(P, sms, st);
    default: return -100;
  }
}

}  // namespace probe
}  // namespace rb200

// returns 0 on success, a CUDA error code, or a negative value: -(CTAs per SM that fit) - 1, -100 for bad arguments
extern "C" int rb200_probe_run(int form, int walk, int minb, int load, int resident, int n_out, int depth, const double* a, double* b, double* c, double* d, long long n,
                               void* stream) {
  using namespace rb200::probe;
  if (n_out != 1 && n_out != 3) return -100;
  if (depth < 2 || depth > 8 || (((uintptr_t)a) & 15u) != 0) return -100;
  Args P;
  P.a = a;
  P.out[0] = b;
  P.out[1] = c;
  P.out[2] = d;
  P.s[0] = 1.5;
  P.s[1] = 2.5;
  P.s[2] = 3.5;
  P.n = n;
  P.n_tiles = (n + TILE - 1) / TILE;
  P.n_out = n_out;
  P.depth = depth;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaStream_t st = (cudaStream_t)stream;
  if (load == 1) {
    if (form != 0 || walk != 0) return -100;
    if (minb < 0 || minb > 8) return -100;
    return launch<0, 0, 2, 1>(P, sms, st, minb == 0, minb, resident);
  }
  if (load != 0 || resident != 0) return -100;
  const int key = form * 2 + walk;
  switch (key) {
    case 0: return by_minb<0, 0>(P, minb, sms, st);
    case 1: return by_minb<0, 1>(P, minb, sms, st);
    case 2: return by_minb<1, 0>(P, minb, sms, st);
    case 3: return by_minb<1, 1>(P, minb, sms, st);
    case 4: return by_minb<2, 0>(P, minb, sms, st);
    case 5: return by_minb<2, 1>(P, minb, sms, st);
    default: return -100;
  }
}
