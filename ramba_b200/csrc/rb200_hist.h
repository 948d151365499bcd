#pragma once
// Binning (rb200_hist.cu): rb200_histogram and rb200_bin_search of include/ramba_b200.h.
#include <cuda_runtime.h>

#include "../../include/ramba_b200.h"
#include "rb200_compact.h"

namespace rb200 {

enum HistForm { HIST_SHARED = 0, HIST_GLOBAL = 1, HIST_SLAB = 2 };

// A validated histogram call: the source (and weights) views, the bin table and the plan every launch and the
// description share.  CTA c covers the C-order positions [c * chunk, min((c + 1) * chunk, n)).
struct HistPlan {
  CompactView src, w;
  bool weighted, vec;
  int src_dtype, w_dtype;
  long long n, B, chunk, ctas;
  int form;
  long long slab, passes;      // bins per pass (B unless SLAB) and passes over the data
  bool table_shared;           // the edge table is staged in shared memory
  long long table_bytes;       // (B + 1) edges (0 for INTEGER)
  long long shared_bytes;      // dynamic shared memory per CTA
  long long scratch_bytes;     // weighted: ctas * slab float64
};

struct SearchPlan {
  CompactView src;
  int src_dtype, tab_dtype, side;
  long long n, n_tab, ctas;
  bool table_shared;
  long long shared_bytes;
};

void make_hist_plan(const rb200_index_view& src, bool weighted, const rb200_bin_table& T, HistPlan* P);
void make_search_plan(const rb200_index_view& src, long long n_tab, int tab_dtype, SearchPlan* P);
cudaError_t launch_histogram(const HistPlan& P, const rb200_bin_table& T, const rb200_index_view* weights, void* out, unsigned long long* bad,
                             void* scratch, cudaStream_t stream);
cudaError_t launch_bin_search(const SearchPlan& P, const void* table, long long* out, cudaStream_t stream);
const char* hist_form_name(int form);

// kernels that stage more than 48 KB of dynamic shared memory must ask for it
template <class K> static inline cudaError_t allow_shared(K kernel, long long smem) {
  if (smem <= 48 * 1024) return cudaSuccess;
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

#ifdef __CUDACC__
// What this lane adds to privatised bin `key` (0xffffffff: no bin) so that the warp adds one per lane that has a bin:
// a warp whose 32 lanes fall into one bin adds 32 once from lane 0 (data skewed into one bin), otherwise every lane
// adds 1.  Every lane of the warp calls it.
__device__ __forceinline__ unsigned warp_bin_share(unsigned key, int lane) {
  const unsigned k0 = __shfl_sync(0xffffffffu, key, 0);
  const bool one = __all_sync(0xffffffffu, key == k0);
  if (key == 0xffffffffu) return 0u;
  return one ? (lane == 0 ? 32u : 0u) : 1u;
}
#endif

}  // namespace rb200
